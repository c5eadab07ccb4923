// Memory-bound row kernels of the encoder: LayerNorm (+GELU) forward / backward with fused residual-gradient add and
// parameter-gradient column reductions, bf16 column sums, GELU-derivative multiply, frame masking, gate (gru_rel_pos),
// relative-position table gather/scatter.  One warp per row, 16-byte vector accesses, warp-shuffle reductions.
#include <algorithm>
#include <type_traits>
#include <type_traits>

#include "../../include/unispeech_b200.h"
#include "common.h"
#include "dropout.cuh"
#include "fp8.cuh"
#include "ptx.cuh"

namespace b200 {

template <int VEC>
struct VecIO;
template <>
struct VecIO<8> {
  static __device__ __forceinline__ void load(const __nv_bfloat16* p, float* v) {
    const uint4 w = *reinterpret_cast<const uint4*>(p);
    const uint32_t u[4] = {w.x, w.y, w.z, w.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float2 f = unpack_bf16x2(u[i]);
      v[2 * i] = f.x;
      v[2 * i + 1] = f.y;
    }
  }
  static __device__ __forceinline__ void store(__nv_bfloat16* p, const float* v) {
    uint4 w;
    w.x = pack_bf16x2(v[0], v[1]); w.y = pack_bf16x2(v[2], v[3]);
    w.z = pack_bf16x2(v[4], v[5]); w.w = pack_bf16x2(v[6], v[7]);
    *reinterpret_cast<uint4*>(p) = w;
  }
};
template <>
struct VecIO<4> {
  static __device__ __forceinline__ void load(const __nv_bfloat16* p, float* v) {
    const uint2 w = *reinterpret_cast<const uint2*>(p);
    const float2 a = unpack_bf16x2(w.x), b = unpack_bf16x2(w.y);
    v[0] = a.x; v[1] = a.y; v[2] = b.x; v[3] = b.y;
  }
  static __device__ __forceinline__ void store(__nv_bfloat16* p, const float* v) {
    uint2 w;
    w.x = pack_bf16x2(v[0], v[1]); w.y = pack_bf16x2(v[2], v[3]);
    *reinterpret_cast<uint2*>(p) = w;
  }
};
template <>
struct VecIO<2> {
  static __device__ __forceinline__ void load(const __nv_bfloat16* p, float* v) {
    const float2 a = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(p));
    v[0] = a.x; v[1] = a.y;
  }
  static __device__ __forceinline__ void store(__nv_bfloat16* p, const float* v) {
    *reinterpret_cast<uint32_t*>(p) = pack_bf16x2(v[0], v[1]);
  }
};

struct RowView {
  long long bs, rs;
  int rows_per_batch;
  // element offset of row r (r < 2^32: every caller's row count is batches x frames); 32-bit division -- the 64-bit one is a
  // ~100-instruction subroutine, which showed in kernels that touch a handful of rows per thread
  __device__ __forceinline__ long long off(long long r) const {
    const unsigned ur = static_cast<unsigned>(r);
    const unsigned b = ur / static_cast<unsigned>(rows_per_batch);
    const unsigned t = ur - b * static_cast<unsigned>(rows_per_batch);
    return static_cast<long long>(b) * bs + static_cast<long long>(t) * rs;
  }
  __device__ __forceinline__ void split(long long r, unsigned& b, unsigned& t) const {
    b = static_cast<unsigned>(r) / static_cast<unsigned>(rows_per_batch);
    t = static_cast<unsigned>(r) - b * static_cast<unsigned>(rows_per_batch);
  }
  __device__ __forceinline__ long long at(unsigned b, unsigned t) const {
    return static_cast<long long>(b) * bs + static_cast<long long>(t) * rs;
  }
};

// V consecutive floats of a 16-byte aligned shared-memory array
template <int V>
__device__ __forceinline__ void smem_load_vec(const float* src, float* v) {
  if constexpr (V % 4 == 0) {
#pragma unroll
    for (int q = 0; q < V / 4; ++q) {
      const float4 t = *reinterpret_cast<const float4*>(src + 4 * q);
      v[4 * q] = t.x; v[4 * q + 1] = t.y; v[4 * q + 2] = t.z; v[4 * q + 3] = t.w;
    }
  } else {
#pragma unroll
    for (int q = 0; q < V; ++q) v[q] = src[q];
  }
}

// ------------------------------------------------------------------------------------------------ LayerNorm forward
// y = (x - mean) * rstd * gamma + beta  [then exact GELU if gelu != 0]; statistics in fp32 (F.layer_norm,
// reference: WavLM/WavLM.py:342,559,666,675; Fp32LayerNorm WavLM/modules.py:30-42 for the conv stack).
// One warp per row; gamma/beta live in shared memory, which keeps the register count at <= 64 and four blocks (32 warps)
// resident per SM: the kernel is latency-, not bandwidth-bound (a row is a chain of loads and two shuffle reductions).
// GATE: also emits the gru_rel_pos gate of the attention that consumes y (WavLM/modules.py:523-533): per head h,
//   (ga, gb) = sigmoid(y_h . wa + ba, y_h . wb + bb),  gate[b,h,t] = ga * (gb * grep_a[h] - 1) + 2,
// where wa / wb are the sums of the first / last four rows of grep_linear.weight and y_h is the STORED (bf16) head slice.
// Needs VEC == 8 (a head's 64 columns = 8 consecutive lanes of one chunk).
struct GateArgs {
  const float* grep_w;  // [8, 64]
  const float* grep_b;  // [8]
  const float* grep_a;  // [H]
  float* gate;          // [B, H, T]
  int H, T;
};

// (D = 1920: 60 values per lane do not fit the 64 registers of four resident blocks; two blocks give 128)
template <int VEC, int NCH, bool GATE, bool GELU>
__global__ void __launch_bounds__(256, 32 * VEC * NCH > 1280 ? 2 : 4) ln_fwd_kernel(const __nv_bfloat16* __restrict__ x, RowView xv,
                                                     const float* __restrict__ gamma, const float* __restrict__ beta,
                                                     __nv_bfloat16* __restrict__ y, RowView yv,
                                                     float* __restrict__ mean_out, float* __restrict__ rstd_out,
                                                     long long rows, float eps, GateArgs ga, const int* __restrict__ valid) {
  pdl_grid_sync();
  constexpr int D = 32 * VEC * NCH;
  constexpr int N = NCH * VEC;
  __shared__ __align__(16) float gs[D], bs[D];
  for (int c = threadIdx.x; c < D; c += blockDim.x) {
    gs[c] = gamma[c];
    bs[c] = beta[c];
  }
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const long long warp_global = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  const long long nwarps = (static_cast<long long>(gridDim.x) * blockDim.x) >> 5;
  float wa[GATE ? 8 : 1], wb[GATE ? 8 : 1], gba = 0.f, gbb = 0.f;
  if constexpr (GATE) {
    static_assert(VEC == 8, "fused gate needs 8 columns per lane");
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int c = (lane & 7) * 8 + j;
      wa[j] = ga.grep_w[c] + ga.grep_w[64 + c] + ga.grep_w[128 + c] + ga.grep_w[192 + c];
      wb[j] = ga.grep_w[256 + c] + ga.grep_w[320 + c] + ga.grep_w[384 + c] + ga.grep_w[448 + c];
    }
    gba = ga.grep_b[0] + ga.grep_b[1] + ga.grep_b[2] + ga.grep_b[3];
    gbb = ga.grep_b[4] + ga.grep_b[5] + ga.grep_b[6] + ga.grep_b[7];
  }
  for (long long r = warp_global; r < rows; r += nwarps) {
    float v[N];
    if (valid != nullptr) {  // ragged batch: a padded frame is written as zeros (finite), nothing is read
      unsigned rb, rt;
      xv.split(r, rb, rt);
      if (static_cast<int>(rt) >= valid[rb]) {
#pragma unroll
        for (int i = 0; i < N; ++i) v[i] = 0.f;
        __nv_bfloat16* yz = y + yv.at(rb, rt);
#pragma unroll
        for (int i = 0; i < NCH; ++i) VecIO<VEC>::store(yz + (i * 32 + lane) * VEC, v + i * VEC);
        if (lane == 0) {
          if (mean_out) mean_out[r] = 0.f;
          if (rstd_out) rstd_out[r] = 0.f;
        }
        if constexpr (GATE) {
          if (lane < ga.H) ga.gate[(static_cast<long long>(rb) * ga.H + lane) * ga.T + rt] = 1.0f;
        }
        continue;
      }
    }
    const __nv_bfloat16* xr = x + xv.off(r);
#pragma unroll
    for (int i = 0; i < NCH; ++i) VecIO<VEC>::load(xr + (i * 32 + lane) * VEC, v + i * VEC);
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < N; ++i) s += v[i];
    const float mean = warp_sum(s) * (1.0f / D);
    float qv = 0.f;
#pragma unroll
    for (int i = 0; i < N; ++i) {
      const float d = v[i] - mean;
      qv += d * d;
    }
    const float rstd = rsqrtf(warp_sum(qv) * (1.0f / D) + eps);
#pragma unroll
    for (int ch = 0; ch < NCH; ++ch) {
      float gg[VEC], bb[VEC];
      smem_load_vec<VEC>(gs + (ch * 32 + lane) * VEC, gg);  // 16-byte loads: scalar ones would be 8-way bank conflicts
      smem_load_vec<VEC>(bs + (ch * 32 + lane) * VEC, bb);
#pragma unroll
      for (int j = 0; j < VEC; ++j) {
        float o = (v[ch * VEC + j] - mean) * rstd * gg[j] + bb[j];
        if (GELU) o = gelu_f(o);
        v[ch * VEC + j] = o;
      }
    }
    __nv_bfloat16* yr = y + yv.off(r);
#pragma unroll
    for (int i = 0; i < NCH; ++i) VecIO<VEC>::store(yr + (i * 32 + lane) * VEC, v + i * VEC);
    if (lane == 0) {
      if (mean_out) mean_out[r] = mean;
      if (rstd_out) rstd_out[r] = rstd;
    }
    if constexpr (GATE) {
      const long long bidx = r / ga.T, t = r % ga.T;
#pragma unroll
      for (int i = 0; i < NCH; ++i) {
        float sa = 0.f, sb = 0.f;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const float yb = __bfloat162float(__float2bfloat16_rn(v[i * 8 + j]));  // what the attention kernel will read
          sa = fmaf(yb, wa[j], sa);
          sb = fmaf(yb, wb[j], sb);
        }
#pragma unroll
        for (int o = 1; o < 8; o <<= 1) {
          sa += __shfl_xor_sync(0xffffffffu, sa, o);
          sb += __shfl_xor_sync(0xffffffffu, sb, o);
        }
        if ((lane & 7) == 0) {
          const int h = i * 4 + (lane >> 3);
          const float g1 = 1.0f / (1.0f + __expf(-(sa + gba)));
          const float g2 = 1.0f / (1.0f + __expf(-(sb + gbb)));
          ga.gate[(bidx * ga.H + h) * ga.T + t] = g1 * (g2 * ga.grep_a[h] - 1.0f) + 2.0f;
        }
      }
    }
  }
}

// LayerNorm forward with an e4m3 output (fp8 inference path, fp8.cuh): ln_fwd_kernel's arithmetic (so y, when written, is
// bit-identical to b200s_layer_norm_fwd's, and the gate is a function of y as in the gate-fused kernels), then the row's amax over the bf16-ROUNDED values, which the warp already holds whole, and
// q = e4m3(y_bf16 * 448 / amax), scale = amax / 448.  y, mean and rstd are optional.  (From D = 512 the row, the amax and the
// gate weights do not fit the 64 registers of four resident blocks without spilling: two blocks.)
struct Fp8Rows {
  uint8_t* q;
  long long bs, rs;  // bytes
  float* scale;      // [rows]
};
template <int VEC>
__device__ __forceinline__ void store_fp8_vec(uint8_t* p, const float* v, float rinv) {
  if constexpr (VEC == 8) *reinterpret_cast<uint2*>(p) = make_uint2(fp8x4(v, rinv), fp8x4(v + 4, rinv));
  else if constexpr (VEC == 4) *reinterpret_cast<uint32_t*>(p) = fp8x4(v, rinv);
  else *reinterpret_cast<uint16_t*>(p) = static_cast<uint16_t>(fp8x2(v[0], v[1], rinv));
}
template <int VEC, int NCH, bool GATE>
__global__ void __launch_bounds__(256, 32 * VEC * NCH >= 512 ? 2 : 4) ln_fwd_fp8_kernel(const __nv_bfloat16* __restrict__ x, RowView xv,
                                                     const float* __restrict__ gamma, const float* __restrict__ beta,
                                                     __nv_bfloat16* __restrict__ y, RowView yv,
                                                     float* __restrict__ mean_out, float* __restrict__ rstd_out,
                                                     long long rows, float eps, GateArgs ga, Fp8Rows f8, const int* __restrict__ valid) {
  pdl_grid_sync();
  constexpr int D = 32 * VEC * NCH;
  constexpr int N = NCH * VEC;
  __shared__ __align__(16) float gs[D], bs[D];
  for (int c = threadIdx.x; c < D; c += blockDim.x) {
    gs[c] = gamma[c];
    bs[c] = beta[c];
  }
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const long long warp_global = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  const long long nwarps = (static_cast<long long>(gridDim.x) * blockDim.x) >> 5;
  float wa[GATE ? 8 : 1], wb[GATE ? 8 : 1], gba = 0.f, gbb = 0.f;
  if constexpr (GATE) {
    static_assert(VEC == 8, "fused gate needs 8 columns per lane");
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int c = (lane & 7) * 8 + j;
      wa[j] = ga.grep_w[c] + ga.grep_w[64 + c] + ga.grep_w[128 + c] + ga.grep_w[192 + c];
      wb[j] = ga.grep_w[256 + c] + ga.grep_w[320 + c] + ga.grep_w[384 + c] + ga.grep_w[448 + c];
    }
    gba = ga.grep_b[0] + ga.grep_b[1] + ga.grep_b[2] + ga.grep_b[3];
    gbb = ga.grep_b[4] + ga.grep_b[5] + ga.grep_b[6] + ga.grep_b[7];
  }
  for (long long r = warp_global; r < rows; r += nwarps) {
    float v[N];
    unsigned rb, rt;
    xv.split(r, rb, rt);
    uint8_t* qr = f8.q + rb * f8.bs + rt * f8.rs;
    if (valid != nullptr && static_cast<int>(rt) >= valid[rb]) {  // ragged batch: a padded frame is written as zeros, nothing read
#pragma unroll
      for (int i = 0; i < N; ++i) v[i] = 0.f;
#pragma unroll
      for (int i = 0; i < NCH; ++i) {
        if (y != nullptr) VecIO<VEC>::store(y + yv.at(rb, rt) + (i * 32 + lane) * VEC, v + i * VEC);
        store_fp8_vec<VEC>(qr + (i * 32 + lane) * VEC, v + i * VEC, 0.f);
      }
      if (lane == 0) {
        f8.scale[r] = 0.f;
        if (mean_out) mean_out[r] = 0.f;
        if (rstd_out) rstd_out[r] = 0.f;
      }
      if constexpr (GATE) {
        if (lane < ga.H) ga.gate[(static_cast<long long>(rb) * ga.H + lane) * ga.T + rt] = 1.0f;
      }
      continue;
    }
    const __nv_bfloat16* xr = x + xv.off(r);
#pragma unroll
    for (int i = 0; i < NCH; ++i) VecIO<VEC>::load(xr + (i * 32 + lane) * VEC, v + i * VEC);
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < N; ++i) s += v[i];
    const float sum = warp_sum(s);
    const float mean = sum * (1.0f / D);
    // x - mean exactly as ln_fwd_kernel's compiled code forms it (so y is bit-identical to b200s_layer_norm_fwd): one FMA with
    // the row sum (the mean is not rounded first), except at D = 1920, where it subtracts the rounded mean.  That form is nvcc's
    // contraction choice for ln_fwd_kernel's `v[i] - mean`, not its source: re-check it (test_layer_norm_fp8) with a new toolchain.
    constexpr bool kFmaMean = D != 1920;
#pragma unroll
    for (int i = 0; i < N; ++i) v[i] = kFmaMean ? fmaf(sum, -(1.0f / D), v[i]) : v[i] - mean;
    float qv = 0.f;
#pragma unroll
    for (int i = 0; i < N; ++i) qv += v[i] * v[i];
    const float rstd = rsqrtf(warp_sum(qv) * (1.0f / D) + eps);
    float amax = 0.f;
#pragma unroll
    for (int ch = 0; ch < NCH; ++ch) {
      float gg[VEC], bb[VEC];
      smem_load_vec<VEC>(gs + (ch * 32 + lane) * VEC, gg);
      smem_load_vec<VEC>(bs + (ch * 32 + lane) * VEC, bb);
#pragma unroll
      for (int j = 0; j < VEC; ++j) {
        const float o = __bfloat162float(__float2bfloat16_rn(v[ch * VEC + j] * rstd * gg[j] + bb[j]));
        v[ch * VEC + j] = o;
        amax = fmaxf(amax, fabsf(o));
      }
    }
    if (y != nullptr) {
      __nv_bfloat16* yr = y + yv.off(r);
#pragma unroll
      for (int i = 0; i < NCH; ++i) VecIO<VEC>::store(yr + (i * 32 + lane) * VEC, v + i * VEC);
    }
    amax = warp_max(amax);
    const float rinv = fp8_row_rinv(amax);
#pragma unroll
    for (int i = 0; i < NCH; ++i) store_fp8_vec<VEC>(qr + (i * 32 + lane) * VEC, v + i * VEC, rinv);
    if (lane == 0) {
      f8.scale[r] = fp8_row_scale(amax);
      if (mean_out) mean_out[r] = mean;
      if (rstd_out) rstd_out[r] = rstd;
    }
    if constexpr (GATE) {
      const long long bidx = r / ga.T, t = r % ga.T;
#pragma unroll
      for (int i = 0; i < NCH; ++i) {
        float sa = 0.f, sb = 0.f;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          sa = fmaf(v[i * 8 + j], wa[j], sa);
          sb = fmaf(v[i * 8 + j], wb[j], sb);
        }
#pragma unroll
        for (int o = 1; o < 8; o <<= 1) {
          sa += __shfl_xor_sync(0xffffffffu, sa, o);
          sb += __shfl_xor_sync(0xffffffffu, sb, o);
        }
        if ((lane & 7) == 0) {
          const int h = i * 4 + (lane >> 3);
          const float g1 = 1.0f / (1.0f + __expf(-(sa + gba)));
          const float g2 = 1.0f / (1.0f + __expf(-(sb + gbb)));
          ga.gate[(bidx * ga.H + h) * ga.T + t] = g1 * (g2 * ga.grep_a[h] - 1.0f) + 2.0f;
        }
      }
    }
  }
}

// Gate-fused forward at wide rows (D = 256 * NW: 512 / 768 / 1024): the row is spread over the NW warps of the block, one
// 16-byte vector per thread, R rows per iteration with all their loads issued up front; mean and variance (two-pass, as above)
// cross the warps through shared memory with one block barrier each.  The gate of a head is an 8-lane affair exactly as in the
// warp-per-row kernel, but all heads of a row are evaluated in parallel (thread t owns columns 8t..8t+7 = head t / 8).
template <int NW, int R>
__global__ void __launch_bounds__(32 * NW) ln_fwd_wide_kernel(const __nv_bfloat16* __restrict__ x, RowView xv,
                                                             const float* __restrict__ gamma, const float* __restrict__ beta,
                                                             __nv_bfloat16* __restrict__ y, RowView yv,
                                                             float* __restrict__ mean_out, float* __restrict__ rstd_out,
                                                             long long rows, float eps, GateArgs ga,
                                                             const int* __restrict__ valid) {
  pdl_grid_sync();
  constexpr int D = 256 * NW;
  const int lane = threadIdx.x & 31;
  const int warp = threadIdx.x >> 5;
  const int c0 = threadIdx.x * 8;
  float g[8], b[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    g[j] = gamma[c0 + j];
    b[j] = beta[c0 + j];
  }
  float wa[8], wb[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const int c = (lane & 7) * 8 + j;
    wa[j] = ga.grep_w[c] + ga.grep_w[64 + c] + ga.grep_w[128 + c] + ga.grep_w[192 + c];
    wb[j] = ga.grep_w[256 + c] + ga.grep_w[320 + c] + ga.grep_w[384 + c] + ga.grep_w[448 + c];
  }
  const float gba = ga.grep_b[0] + ga.grep_b[1] + ga.grep_b[2] + ga.grep_b[3];
  const float gbb = ga.grep_b[4] + ga.grep_b[5] + ga.grep_b[6] + ga.grep_b[7];
  const float a_h = ga.grep_a[threadIdx.x >> 3];
  __shared__ float red[2][NW][R];
  for (long long r0 = static_cast<long long>(blockIdx.x) * R; r0 < rows; r0 += static_cast<long long>(gridDim.x) * R) {
    uint4 raw[R];
    unsigned rb[R], rt[R];
    bool dead[R];  // ragged batch: padded frame -> zeros out, nothing read
#pragma unroll
    for (int i = 0; i < R; ++i) {
      const long long r = r0 + i;
      xv.split(r < rows ? r : 0, rb[i], rt[i]);
      dead[i] = valid != nullptr && r < rows && static_cast<int>(rt[i]) >= valid[rb[i]];
      raw[i] = (r < rows && !dead[i]) ? *reinterpret_cast<const uint4*>(x + xv.at(rb[i], rt[i]) + c0) : make_uint4(0u, 0u, 0u, 0u);
    }
    float v[R][8], s[R];
#pragma unroll
    for (int i = 0; i < R; ++i) {
      const uint32_t u[4] = {raw[i].x, raw[i].y, raw[i].z, raw[i].w};
      s[i] = 0.f;
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const float2 f = unpack_bf16x2(u[k]);
        v[i][2 * k] = f.x;
        v[i][2 * k + 1] = f.y;
        s[i] += f.x + f.y;
      }
    }
#pragma unroll
    for (int i = 0; i < R; ++i) s[i] = warp_sum(s[i]);
    if (lane == 0) {
#pragma unroll
      for (int i = 0; i < R; ++i) red[0][warp][i] = s[i];
    }
    __syncthreads();
    float mean[R], rstd[R];
#pragma unroll
    for (int i = 0; i < R; ++i) {
      float t = 0.f;
#pragma unroll
      for (int w = 0; w < NW; ++w) t += red[0][w][i];
      mean[i] = t * (1.0f / D);
      float q = 0.f;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float d = v[i][j] - mean[i];
        q = fmaf(d, d, q);
      }
      s[i] = warp_sum(q);
    }
    if (lane == 0) {
#pragma unroll
      for (int i = 0; i < R; ++i) red[1][warp][i] = s[i];
    }
    __syncthreads();
#pragma unroll
    for (int i = 0; i < R; ++i) {
      float t = 0.f;
#pragma unroll
      for (int w = 0; w < NW; ++w) t += red[1][w][i];
      rstd[i] = rsqrtf(t * (1.0f / D) + eps);
    }
#pragma unroll
    for (int i = 0; i < R; ++i) {
      const long long r = r0 + i;
      uint32_t ou[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const float o0 = (v[i][2 * k] - mean[i]) * rstd[i] * g[2 * k] + b[2 * k];
        const float o1 = (v[i][2 * k + 1] - mean[i]) * rstd[i] * g[2 * k + 1] + b[2 * k + 1];
        ou[k] = dead[i] ? 0u : pack_bf16x2(o0, o1);
      }
      if (r < rows) {
        *reinterpret_cast<uint4*>(y + yv.at(rb[i], rt[i]) + c0) = make_uint4(ou[0], ou[1], ou[2], ou[3]);
        if (threadIdx.x == 0) {
          if (mean_out) mean_out[r] = dead[i] ? 0.f : mean[i];
          if (rstd_out) rstd_out[r] = dead[i] ? 0.f : rstd[i];
        }
      }
      float sa = 0.f, sb = 0.f;
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const float2 yb = unpack_bf16x2(ou[k]);  // what the attention kernel will read
        sa = fmaf(yb.x, wa[2 * k], sa);
        sa = fmaf(yb.y, wa[2 * k + 1], sa);
        sb = fmaf(yb.x, wb[2 * k], sb);
        sb = fmaf(yb.y, wb[2 * k + 1], sb);
      }
#pragma unroll
      for (int o = 1; o < 8; o <<= 1) {
        sa += __shfl_xor_sync(0xffffffffu, sa, o);
        sb += __shfl_xor_sync(0xffffffffu, sb, o);
      }
      if ((lane & 7) == 0 && r < rows) {
        const long long bidx = rb[i], t = rt[i];  // (the views have T rows per batch)
        const float g1 = 1.0f / (1.0f + __expf(-(sa + gba)));
        const float g2 = 1.0f / (1.0f + __expf(-(sb + gbb)));
        ga.gate[(bidx * ga.H + (threadIdx.x >> 3)) * ga.T + t] = dead[i] ? 1.0f : g1 * (g2 * a_h - 1.0f) + 2.0f;
      }
    }
  }
}

template <typename... Args>
static int launch_ln_fwd_wide(int D, long long rows, cudaStream_t st, Args... args) {
  constexpr int R = 4;
  auto go = [&](auto nw) {
    constexpr int NW = decltype(nw)::value;
    auto kern = ln_fwd_wide_kernel<NW, R>;
    static const int cap = resident_grid(kern, 32 * NW);
    const int grid = static_cast<int>(std::min<long long>(ceil_div_ll(rows, R), cap));
    B200_CHECK_CUDA(launch_pdl(kern, dim3(grid), dim3(32 * NW), 0, st, args...));
    return 0;
  };
  const int rc = D == 512 ? go(std::integral_constant<int, 2>{}) : D == 768 ? go(std::integral_constant<int, 3>{})
                                                                           : go(std::integral_constant<int, 4>{});
  if (rc) return rc;
  B200_CHECK_LAUNCH();
  return 0;
}

// ------------------------------------------------------------------------------------------------ LayerNorm backward
// dz = dy * gelu'(gamma*xhat+beta) if gelu else dy;  dxhat = dz*gamma
// dx = rstd * (dxhat - mean(dxhat) - xhat*mean(dxhat*xhat)) [+ dres];  dgamma += sum_rows dz*xhat; dbeta += sum_rows dz
// optional colsum += sum_rows dx (as stored, bf16-rounded) -- the bias gradient of the producer of x.
// dst[0..V) += v[0..V) on a lane-private shared-memory slice, with 16-byte accesses where possible (conflict-free: consecutive
// lanes own consecutive V-float segments)
template <int V>
__device__ __forceinline__ void smem_add_vec(float* dst, const float* v) {
  if constexpr (V % 4 == 0) {
#pragma unroll
    for (int q = 0; q < V / 4; ++q) {
      float4 t = *reinterpret_cast<float4*>(dst + 4 * q);
      t.x += v[4 * q]; t.y += v[4 * q + 1]; t.z += v[4 * q + 2]; t.w += v[4 * q + 3];
      *reinterpret_cast<float4*>(dst + 4 * q) = t;
    }
  } else {
#pragma unroll
    for (int q = 0; q < V; ++q) dst[q] += v[q];
  }
}

// Bank-conflict-free placement of a [D] fp32 row whose lanes own VEC consecutive columns: with VEC = 8 the natural layout puts
// the lanes 32 bytes apart, so a 128-bit access by a warp touches every other 16-byte slot and runs at half rate (ncu: 2.6 bank
// conflicts per shared request in the LayerNorm backward, which made it MIO-bound at 20 % of the HBM peak).  Here the two
// float4 halves of a lane's 8 columns go to two separate 512-byte planes, lanes 16 bytes apart.
template <int VEC>
__device__ __forceinline__ int perm_col(int c) {
  if constexpr (VEC == 8) {
    const int ch = c >> 8, rem = c & 255, lane = rem >> 3, j = rem & 7;
    return ((ch * 2 + (j >> 2)) * 32 + lane) * 4 + (j & 3);
  } else {
    return c;
  }
}
template <int VEC>
__device__ __forceinline__ void smem_load_perm(const float* base, int ch, int lane, float* v) {
  if constexpr (VEC == 8) {
#pragma unroll
    for (int k = 0; k < 2; ++k) {
      const float4 t = *reinterpret_cast<const float4*>(base + ((ch * 2 + k) * 32 + lane) * 4);
      v[4 * k] = t.x; v[4 * k + 1] = t.y; v[4 * k + 2] = t.z; v[4 * k + 3] = t.w;
    }
  } else {
    smem_load_vec<VEC>(base + (ch * 32 + lane) * VEC, v);
  }
}
template <int VEC>
__device__ __forceinline__ void smem_add_perm(float* base, int ch, int lane, const float* v) {
  if constexpr (VEC == 8) {
#pragma unroll
    for (int k = 0; k < 2; ++k) {
      float4* p = reinterpret_cast<float4*>(base + ((ch * 2 + k) * 32 + lane) * 4);
      float4 t = *p;
      t.x += v[4 * k]; t.y += v[4 * k + 1]; t.z += v[4 * k + 2]; t.w += v[4 * k + 3];
      *p = t;
    }
  } else {
    smem_add_vec<VEC>(base + (ch * 32 + lane) * VEC, v);
  }
}

// (D = 1920: one resident block, which its 195 KB of column partials allow anyway, so 60 values per lane fit in registers)
template <int VEC, int NCH>
__global__ void __launch_bounds__(256, 32 * VEC * NCH > 1280 ? 1 : 2) ln_bwd_kernel(const __nv_bfloat16* __restrict__ dy, RowView dyv,
                                                        const __nv_bfloat16* __restrict__ x, RowView xv,
                                                        const float* __restrict__ mean_in, const float* __restrict__ rstd_in,
                                                        const float* __restrict__ gamma, const float* __restrict__ beta,
                                                        const __nv_bfloat16* __restrict__ dres, RowView dresv,
                                                        __nv_bfloat16* __restrict__ dx, RowView dxv,
                                                        float* __restrict__ dgamma, float* __restrict__ dbeta,
                                                        float* __restrict__ colsum, long long rows, int gelu,
                                                        const int* __restrict__ valid) {
  pdl_grid_sync();
  constexpr int D = 32 * VEC * NCH;
  constexpr int N = NCH * VEC;
  // The per-warp column partials (d gamma, d beta, column sums of dx) live in SHARED memory, not in 3*N registers per lane:
  // the kernel is latency-bound (a row is loads -> two shuffle reductions -> store), and at 226 registers only one block
  // (8 warps) fitted an SM.  Layout: acc[q][warp][D] fp32, then gamma[D], beta[D].
  extern __shared__ __align__(16) float ln_smem[];
  float* acc = ln_smem;
  float* gs = ln_smem + 3 * 8 * D;
  float* bs = gs + D;
  const int lane = threadIdx.x & 31;
  const int warp = threadIdx.x >> 5;
  for (int c = threadIdx.x; c < 3 * 8 * D; c += blockDim.x) acc[c] = 0.f;
  for (int c = threadIdx.x; c < D; c += blockDim.x) {
    gs[perm_col<VEC>(c)] = gamma[c];
    bs[perm_col<VEC>(c)] = gelu ? beta[c] : 0.f;
  }
  __syncthreads();
  const long long warp_global = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  const long long nwarps = (static_cast<long long>(gridDim.x) * blockDim.x) >> 5;
  float* my_g = acc + (0 * 8 + warp) * D;
  float* my_b = acc + (1 * 8 + warp) * D;
  float* my_c = acc + (2 * 8 + warp) * D;
  const bool want_gb = dgamma != nullptr || dbeta != nullptr;
  const bool want_c = colsum != nullptr;

  // The kernel is latency-bound (a row is loads -> two shuffle reductions -> store, 16 warps per SM): the NEXT row's x vectors and
  // statistics are requested (raw, still packed as bf16) before the current row is touched, so each warp keeps 1.5 rows of loads
  // in flight (prefetching dy as well does not fit the 128-register budget at D = 1024 without spilling).
  using RawVec = typename std::conditional<VEC == 8, uint4, typename std::conditional<VEC == 4, uint2, uint32_t>::type>::type;
  RawVec nx[NCH];
  float nmean = 0.f, nrstd = 0.f;
  auto fetch = [&](long long r) {
    const __nv_bfloat16* xr = x + xv.off(r);
#pragma unroll
    for (int i = 0; i < NCH; ++i) nx[i] = *reinterpret_cast<const RawVec*>(xr + (i * 32 + lane) * VEC);
    nmean = mean_in[r];
    nrstd = rstd_in[r];
  };
  // ragged batch: the gradient of a padded frame is zero by construction -- its dx row is written as zeros, nothing is read
  auto dead = [&](long long r) {
    if (valid == nullptr) return false;
    unsigned rb, rt;
    xv.split(r, rb, rt);
    return static_cast<int>(rt) >= valid[rb];
  };
  if (warp_global < rows && !dead(warp_global)) fetch(warp_global);
  for (long long r = warp_global; r < rows; r += nwarps) {
    float xh[N], dz[N];
    if (dead(r)) {
#pragma unroll
      for (int i = 0; i < VEC; ++i) dz[i] = 0.f;
      __nv_bfloat16* oz = dx + dxv.off(r);
#pragma unroll
      for (int i = 0; i < NCH; ++i) VecIO<VEC>::store(oz + (i * 32 + lane) * VEC, dz);
      if (r + nwarps < rows && !dead(r + nwarps)) fetch(r + nwarps);
      continue;
    }
    const __nv_bfloat16* dr = dy + dyv.off(r);
#pragma unroll
    for (int i = 0; i < NCH; ++i) {
      VecIO<VEC>::load(dr + (i * 32 + lane) * VEC, dz + i * VEC);
      const uint32_t* u = reinterpret_cast<const uint32_t*>(&nx[i]);
#pragma unroll
      for (int k = 0; k < VEC / 2; ++k) {
        const float2 f = unpack_bf16x2(u[k]);
        xh[i * VEC + 2 * k] = f.x;
        xh[i * VEC + 2 * k + 1] = f.y;
      }
    }
    const float mean = nmean, rstd = nrstd;
    if (r + nwarps < rows && !dead(r + nwarps)) fetch(r + nwarps);
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int ch = 0; ch < NCH; ++ch) {
      float pg[VEC], pb[VEC], gg[VEC], bb[VEC];
      smem_load_perm<VEC>(gs, ch, lane, gg);
      if (gelu) smem_load_perm<VEC>(bs, ch, lane, bb);
#pragma unroll
      for (int j = 0; j < VEC; ++j) {
        const int i = ch * VEC + j;
        xh[i] = (xh[i] - mean) * rstd;
        const float gi = gg[j];
        if (gelu) dz[i] *= gelu_grad_f(gi * xh[i] + bb[j]);
        pg[j] = dz[i] * xh[i];
        pb[j] = dz[i];
        const float dxh = dz[i] * gi;
        dz[i] = dxh;
        s1 += dxh;
        s2 += dxh * xh[i];
      }
      if (want_gb) smem_add_perm<VEC>(my_g, ch, lane, pg), smem_add_perm<VEC>(my_b, ch, lane, pb);
    }
    s1 = warp_sum(s1) * (1.0f / D);
    s2 = warp_sum(s2) * (1.0f / D);
    if (dres != nullptr) {
      const __nv_bfloat16* rr = dres + dresv.off(r);
      float o[VEC];
#pragma unroll
      for (int i = 0; i < NCH; ++i) {
        VecIO<VEC>::load(rr + (i * 32 + lane) * VEC, o);
#pragma unroll
        for (int j = 0; j < VEC; ++j) dz[i * VEC + j] = o[j] + rstd * (dz[i * VEC + j] - s1 - xh[i * VEC + j] * s2);
      }
    } else {
#pragma unroll
      for (int i = 0; i < N; ++i) dz[i] = rstd * (dz[i] - s1 - xh[i] * s2);
    }
    if (want_c) {
#pragma unroll
      for (int ch = 0; ch < NCH; ++ch) {
        float pc[VEC];
#pragma unroll
        for (int j = 0; j < VEC; ++j) pc[j] = __bfloat162float(__float2bfloat16_rn(dz[ch * VEC + j]));
        smem_add_perm<VEC>(my_c, ch, lane, pc);
      }
    }
    __nv_bfloat16* outr = dx + dxv.off(r);
#pragma unroll
    for (int i = 0; i < NCH; ++i) VecIO<VEC>::store(outr + (i * 32 + lane) * VEC, dz + i * VEC);
  }

  // block reduction of the per-warp column partials
  __syncthreads();
  const int nw = blockDim.x >> 5;
  for (int c = threadIdx.x; c < D; c += blockDim.x) {
    float sg = 0.f, sb = 0.f, sc = 0.f;
    const int pc = perm_col<VEC>(c);
    for (int w = 0; w < nw; ++w) {
      sg += acc[(0 * 8 + w) * D + pc];
      sb += acc[(1 * 8 + w) * D + pc];
      sc += acc[(2 * 8 + w) * D + pc];
    }
    if (dgamma != nullptr) atomicAdd(dgamma + c, sg);
    if (dbeta != nullptr) atomicAdd(dbeta + c, sb);
    if (colsum != nullptr) atomicAdd(colsum + c, sc);
  }
}

// blocks of `threads` threads of kernel `k` that fit the chip at once (a grid-stride kernel gains nothing from more)
template <typename K>
static int resident_grid(K k, int threads) {
  int per_sm = 1;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k, threads, 0) != cudaSuccess || per_sm < 1) per_sm = 1;
  return per_sm * sm_count();
}

template <typename F>
static int dispatch_width(int D, F&& f) {
  switch (D) {
    case 64: return f(std::integral_constant<int, 2>{}, std::integral_constant<int, 1>{});
    case 128: return f(std::integral_constant<int, 4>{}, std::integral_constant<int, 1>{});
    case 256: return f(std::integral_constant<int, 8>{}, std::integral_constant<int, 1>{});
    case 512: return f(std::integral_constant<int, 8>{}, std::integral_constant<int, 2>{});
    case 768: return f(std::integral_constant<int, 8>{}, std::integral_constant<int, 3>{});
    case 1024: return f(std::integral_constant<int, 8>{}, std::integral_constant<int, 4>{});
    case 1280: return f(std::integral_constant<int, 8>{}, std::integral_constant<int, 5>{});
    case 1920: return f(std::integral_constant<int, 4>{}, std::integral_constant<int, 15>{});  // not 32 x 8 x n
    default:
      set_last_error("row kernels support widths 64/128/256/512/768/1024/1280/1920, got %d", D);
      return -1;
  }
}

// one row per warp and iteration, 8 warps per block, four resident blocks per SM
static int ln_fwd_grid(long long rows) {
  long long blocks = ceil_div_ll(rows, 8);
  const long long cap = static_cast<long long>(sm_count()) * 4;
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  return static_cast<int>(blocks);
}

static int row_grid(long long rows, int warps_per_block) {
  long long blocks = ceil_div_ll(rows, warps_per_block);
  const long long cap = static_cast<long long>(sm_count()) * 8;
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  return static_cast<int>(blocks);
}

// ------------------------------------------------------------------------------------------------ column sums
// colsum[c] += sum_rows x[r, c]   (bias gradients); x bf16 [rows, N] with batch/row strides.
__global__ void __launch_bounds__(256) colsum_kernel(const __nv_bfloat16* __restrict__ x, RowView xv, int N,
                                                     long long rows, float* __restrict__ out, const int* __restrict__ valid) {
  pdl_grid_sync();
  // block: a strip of 256 columns (32 lanes x 8 columns, 16-byte loads) x 8 row lanes; rows strided over blockIdx.y
  const int lane = threadIdx.x & 31;
  const int c = blockIdx.x * 256 + lane * 8;
  const int rl = threadIdx.x >> 5;  // 0..7
  float a[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) a[i] = 0.f;
  if (c < N) {
    const long long step = static_cast<long long>(gridDim.y) * 8;
#pragma unroll 4
    for (long long r = static_cast<long long>(blockIdx.y) * 8 + rl; r < rows; r += step) {
      float v[8];
      if (valid != nullptr) {  // ragged batch: padded frames hold zeros
        unsigned rb, rt;
        xv.split(r, rb, rt);
        if (static_cast<int>(rt) >= valid[rb]) continue;
      }
      VecIO<8>::load(x + xv.off(r) + c, v);
#pragma unroll
      for (int i = 0; i < 8; ++i) a[i] += v[i];
    }
  }
  __shared__ float red[8][256];
#pragma unroll
  for (int i = 0; i < 8; ++i) red[rl][lane * 8 + i] = a[i];
  __syncthreads();
  float s = 0.f;
#pragma unroll
  for (int w = 0; w < 8; ++w) s += red[w][threadIdx.x];
  const int cc = blockIdx.x * 256 + threadIdx.x;
  if (cc < N) atomicAdd(out + cc, s);
}

// ------------------------------------------------------------------------------------------------ dgelu multiply
// out = dy * gelu'(pre)  (bf16), optional colsum of the stored values.  Used for the pos_conv backward
// (x + gelu(conv(x)): WavLM/WavLM.py:577-579) where the product must land in a zero-padded buffer.
__global__ void __launch_bounds__(256) dgelu_mul_kernel(const __nv_bfloat16* __restrict__ dy, RowView dyv,
                                                        const __nv_bfloat16* __restrict__ pre, RowView prev,
                                                        __nv_bfloat16* __restrict__ out, RowView outv, int N,
                                                        long long rows, float* __restrict__ colsum, int pre_is_grad) {
  pdl_grid_sync();
  const int c = blockIdx.x * 64 + (threadIdx.x & 31) * 2;
  const int rl = threadIdx.x >> 5;
  float a0 = 0.f, a1 = 0.f;
  if (c < N) {
    for (long long r = static_cast<long long>(blockIdx.y) * 8 + rl; r < rows; r += static_cast<long long>(gridDim.y) * 8) {
      const float2 d = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(dy + dyv.off(r) + c));
      const float2 p = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(pre + prev.off(r) + c));
      const uint32_t w = pre_is_grad ? pack_bf16x2(d.x * p.x, d.y * p.y)
                                     : pack_bf16x2(d.x * gelu_grad_f(p.x), d.y * gelu_grad_f(p.y));
      *reinterpret_cast<uint32_t*>(out + outv.off(r) + c) = w;
      const float2 f = unpack_bf16x2(w);
      a0 += f.x;
      a1 += f.y;
    }
  }
  if (colsum == nullptr) return;
  __shared__ float red[8][64];
  red[rl][(threadIdx.x & 31) * 2] = a0;
  red[rl][(threadIdx.x & 31) * 2 + 1] = a1;
  __syncthreads();
  if (threadIdx.x < 64) {
    float s = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) s += red[w][threadIdx.x];
    const int cc = blockIdx.x * 64 + threadIdx.x;
    if (cc < N) atomicAdd(colsum + cc, s);
  }
}

// ------------------------------------------------------------------------------------------------ dropout
// y = [res +] dropout(x): nn.Dropout / F.dropout of the transformer stack (WavLM/WavLM.py:350,584,702,711,713,726,736,738).
// The mask is a pure function of (key, logical row, column) (dropout.cuh), so the backward pass is the same kernel applied to
// the incoming gradient with the same key (res = null).  8 bf16 per thread, grid-stride over 16-byte vectors; x == y is allowed.
template <bool HAS_RES>
__global__ void __launch_bounds__(256) dropout_rows_kernel(const __nv_bfloat16* x, RowView xv, const __nv_bfloat16* res,
                                                           RowView rv, __nv_bfloat16* y, RowView yv, int N,
                                                           unsigned total_vecs, uint32_t k0, uint32_t k1, uint32_t thr_hi,
                                                           float rp) {
  pdl_grid_sync();
  const unsigned vec_per_row = static_cast<unsigned>(N) >> 3;
  for (unsigned v = blockIdx.x * 256u + threadIdx.x; v < total_vecs; v += gridDim.x * 256u) {
    const unsigned row = v / vec_per_row;
    const unsigned c = (v - row * vec_per_row) << 3;
    float a[8];
    VecIO<8>::load(x + xv.off(row) + c, a);
    const uint32_t ctr0 = (row * static_cast<uint32_t>(N) + c) >> 1;
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const uint32_t bits = drop_bits(k0, k1, ctr0 + q);
      a[2 * q] = drop_keep_lo(bits, thr_hi) ? a[2 * q] * rp : 0.f;
      a[2 * q + 1] = drop_keep_hi(bits, thr_hi) ? a[2 * q + 1] * rp : 0.f;
    }
    if (HAS_RES) {
      float b[8];
      VecIO<8>::load(res + rv.off(row) + c, b);
#pragma unroll
      for (int q = 0; q < 8; ++q) a[q] += b[q];
    }
    VecIO<8>::store(y + yv.off(row) + c, a);
  }
}

// ------------------------------------------------------------------------------------------------ GradMultiply / features_pen
// features_pen = mean(features^2) over the valid rows (src/fairseq/models/wavlm/wavlm.py:484; WavLM/WavLM.py has no penalty):
// one pass, fp64 accumulator on the device (no host synchronisation).
__global__ void __launch_bounds__(256) sumsq_rows_kernel(const __nv_bfloat16* __restrict__ x, RowView xv, int N,
                                                         unsigned total_vecs, double* __restrict__ out) {
  pdl_grid_sync();
  const unsigned vec_per_row = static_cast<unsigned>(N) >> 3;
  float acc = 0.f;
  for (unsigned v = blockIdx.x * 256u + threadIdx.x; v < total_vecs; v += gridDim.x * 256u) {
    const unsigned row = v / vec_per_row;
    const unsigned c = (v - row * vec_per_row) << 3;
    float a[8];
    VecIO<8>::load(x + xv.off(row) + c, a);
#pragma unroll
    for (int q = 0; q < 8; ++q) acc = fmaf(a[q], a[q], acc);
  }
  double d = static_cast<double>(warp_sum(acc));
  __shared__ double red[8];
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = d;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
    for (int w = 0; w < 8; ++w) t += red[w];
    atomicAdd(out, t);
  }
}

// Backward of GradMultiply.apply(features, scale) (WavLM/modules.py:60-69; WavLM/WavLM.py:333-336) fused with the gradient of the
// feature penalty taken on its output (fairseq wavlm.py:477-484):   g <- scale * (g + coef * x),   coef = *pen_grad * pen_mul
// (pen_grad: the upstream gradient of the penalty scalar, a DEVICE float, or NULL for none).  In place on g.
__global__ void __launch_bounds__(256) grad_multiply_kernel(__nv_bfloat16* __restrict__ g, RowView gv,
                                                            const __nv_bfloat16* __restrict__ x, RowView xv, int N,
                                                            unsigned total_vecs, float scale, const float* __restrict__ pen_grad,
                                                            float pen_mul) {
  pdl_grid_sync();
  const unsigned vec_per_row = static_cast<unsigned>(N) >> 3;
  const float coef = (pen_grad != nullptr) ? (*pen_grad) * pen_mul : 0.f;
  for (unsigned v = blockIdx.x * 256u + threadIdx.x; v < total_vecs; v += gridDim.x * 256u) {
    const unsigned row = v / vec_per_row;
    const unsigned c = (v - row * vec_per_row) << 3;
    float a[8];
    VecIO<8>::load(g + gv.off(row) + c, a);
    if (pen_grad != nullptr) {
      float b[8];
      VecIO<8>::load(x + xv.off(row) + c, b);
#pragma unroll
      for (int q = 0; q < 8; ++q) a[q] = fmaf(coef, b[q], a[q]);
    }
#pragma unroll
    for (int q = 0; q < 8; ++q) a[q] *= scale;
    VecIO<8>::store(g + gv.off(row) + c, a);
  }
}

// ------------------------------------------------------------------------------------------------ frame masking
// x[b,t,:] = 0 where pad[b,t];  = mask_emb where mask[b,t] and not pad   (apply_mask WavLM/WavLM.py:285-286, then
// x[padding_mask] = 0 WavLM/WavLM.py:574-575).  In place on a [B,T,D] view.
// CHAN: channel masking, the second half of apply_mask (WavLM/WavLM.py:288-307): x[b,:,c] = 0 where chan[b,c], applied after
// the mask_emb line, so a time-masked frame loses its masked channels too.  Every unpadded row is visited then; a bf16 pair
// is cleared by bit masking, so the values that survive are the input's bits.
__device__ __forceinline__ uint32_t chan_keep_bits(uint16_t cm) {  // cm: chan[c] in the low byte, chan[c + 1] in the high byte
  return ((cm & 0x00FFu) ? 0xFFFF0000u : 0xFFFFFFFFu) & ((cm & 0xFF00u) ? 0x0000FFFFu : 0xFFFFFFFFu);
}

template <bool CHAN>
__global__ void __launch_bounds__(256) frame_mask_fwd_kernel(__nv_bfloat16* __restrict__ x, RowView xv, int D,
                                                             long long rows, const uint8_t* __restrict__ mask,
                                                             const uint8_t* __restrict__ pad,
                                                             const float* __restrict__ mask_emb,
                                                             const uint8_t* __restrict__ chan) {
  pdl_grid_sync();
  const int lane = threadIdx.x & 31;
  const long long warp_global = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  const long long nwarps = (static_cast<long long>(gridDim.x) * blockDim.x) >> 5;
  for (long long r = warp_global; r < rows; r += nwarps) {
    const bool p = pad != nullptr && pad[r] != 0;
    const bool m = mask != nullptr && mask[r] != 0;
    if constexpr (!CHAN) {
      if (!p && !m) continue;
      __nv_bfloat16* xr = x + xv.off(r);
      for (int c = lane * 2; c < D; c += 64) {
        const uint32_t w = p ? 0u : pack_bf16x2(mask_emb[c], mask_emb[c + 1]);
        *reinterpret_cast<uint32_t*>(xr + c) = w;
      }
    } else {
      __nv_bfloat16* xr = x + xv.off(r);
      const uint8_t* cr = chan + static_cast<long long>(static_cast<unsigned>(r) / static_cast<unsigned>(xv.rows_per_batch)) * D;
      for (int c = lane * 2; c < D; c += 64) {
        uint32_t* px = reinterpret_cast<uint32_t*>(xr + c);
        if (p) {
          *px = 0u;
          continue;
        }
        const uint16_t cm = *reinterpret_cast<const uint16_t*>(cr + c);
        if (!m && cm == 0) continue;  // untouched pair
        const uint32_t w = m ? pack_bf16x2(mask_emb[c], mask_emb[c + 1]) : *px;
        *px = w & chan_keep_bits(cm);
      }
    }
  }
}
// backward: d mask_emb += sum over masked & unpadded rows of dx;  dx rows that were overwritten get zero gradient.
// CHAN: entries of masked channels were overwritten too: their dx is zero and they add nothing to d mask_emb.
template <bool CHAN>
__global__ void __launch_bounds__(256) frame_mask_bwd_kernel(__nv_bfloat16* __restrict__ dx, RowView xv, int D,
                                                             long long rows, const uint8_t* __restrict__ mask,
                                                             const uint8_t* __restrict__ pad,
                                                             float* __restrict__ dmask_emb,
                                                             const uint8_t* __restrict__ chan) {
  pdl_grid_sync();
  const int lane = threadIdx.x & 31;
  const long long warp_global = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  const long long nwarps = (static_cast<long long>(gridDim.x) * blockDim.x) >> 5;
  // per-warp register partials of d mask_emb (lane owns columns lane*2 + 64*i): one atomic per column per warp at the end
  // instead of one per masked row (65 % of the rows hit the same D addresses)
  constexpr int kMaxIter = 32;  // D <= 2048
  float acc[kMaxIter][2];
#pragma unroll
  for (int i = 0; i < kMaxIter; ++i) acc[i][0] = acc[i][1] = 0.f;
  for (long long r = warp_global; r < rows; r += nwarps) {
    const bool p = pad != nullptr && pad[r] != 0;
    const bool m = mask != nullptr && mask[r] != 0;
    if constexpr (!CHAN) {
      if (!p && !m) continue;
      __nv_bfloat16* xr = dx + xv.off(r);
#pragma unroll
      for (int i = 0; i < kMaxIter; ++i) {
        const int c = lane * 2 + 64 * i;
        if (c < D) {
          if (!p) {
            const float2 f = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(xr + c));
            acc[i][0] += f.x;
            acc[i][1] += f.y;
          }
          *reinterpret_cast<uint32_t*>(xr + c) = 0u;
        }
      }
    } else {
      __nv_bfloat16* xr = dx + xv.off(r);
      const uint8_t* cr = chan + static_cast<long long>(static_cast<unsigned>(r) / static_cast<unsigned>(xv.rows_per_batch)) * D;
#pragma unroll
      for (int i = 0; i < kMaxIter; ++i) {
        const int c = lane * 2 + 64 * i;
        if (c < D) {
          uint32_t* px = reinterpret_cast<uint32_t*>(xr + c);
          const uint16_t cm = p ? 0xFFFFu : *reinterpret_cast<const uint16_t*>(cr + c);
          if (m && !p) {
            const float2 f = unpack_bf16x2(*px);
            acc[i][0] += (cm & 0x00FFu) ? 0.f : f.x;
            acc[i][1] += (cm & 0xFF00u) ? 0.f : f.y;
          }
          if (m || p) {
            *px = 0u;
          } else if (cm != 0) {
            *px &= chan_keep_bits(cm);
          }
        }
      }
    }
  }
  if (dmask_emb != nullptr) {
#pragma unroll
    for (int i = 0; i < kMaxIter; ++i) {
      const int c = lane * 2 + 64 * i;
      if (c < D && (acc[i][0] != 0.f || acc[i][1] != 0.f)) {
        atomicAdd(dmask_emb + c, acc[i][0]);
        atomicAdd(dmask_emb + c + 1, acc[i][1]);
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------ gru_rel_pos gate
// gate[b,h,t] = ga*(gb*grep_a[h] - 1) + 2, (ga,gb) = sigmoid(sum of the first / last 4 outputs of grep_linear applied to
// the raw 64-wide head slice of the layer input)  (WavLM/modules.py:523-533).  wa/wb are the pre-summed weight rows.
__global__ void __launch_bounds__(256) gate_fwd_kernel(const __nv_bfloat16* __restrict__ x, RowView xv, int H, int T,
                                                       long long rows, const float* __restrict__ grep_w,
                                                       const float* __restrict__ grep_b, const float* __restrict__ grep_a,
                                                       float* __restrict__ gate) {
  pdl_grid_sync();
  const int lane = threadIdx.x & 31;
  const long long warp_global = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  const long long nwarps = (static_cast<long long>(gridDim.x) * blockDim.x) >> 5;
  float wa0 = 0.f, wa1 = 0.f, wb0 = 0.f, wb1 = 0.f, ba = 0.f, bb = 0.f;
#pragma unroll
  for (int o = 0; o < 4; ++o) {
    wa0 += grep_w[o * 64 + lane * 2];
    wa1 += grep_w[o * 64 + lane * 2 + 1];
    wb0 += grep_w[(o + 4) * 64 + lane * 2];
    wb1 += grep_w[(o + 4) * 64 + lane * 2 + 1];
    ba += grep_b[o];
    bb += grep_b[o + 4];
  }
  for (long long r = warp_global; r < rows; r += nwarps) {
    const __nv_bfloat16* xr = x + xv.off(r);
    const unsigned ub = static_cast<unsigned>(r) / static_cast<unsigned>(T);
    const long long b = ub, t = static_cast<unsigned>(r) - ub * static_cast<unsigned>(T);
#pragma unroll 4
    for (int h = 0; h < H; ++h) {
      const float2 f = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(xr + h * 64 + lane * 2));
      const float sa = warp_sum(f.x * wa0 + f.y * wa1) + ba;
      const float sb = warp_sum(f.x * wb0 + f.y * wb1) + bb;
      if (lane == 0) {
        const float ga = 1.0f / (1.0f + __expf(-sa));
        const float gb = 1.0f / (1.0f + __expf(-sb));
        gate[(b * H + h) * T + t] = ga * (gb * grep_a[h] - 1.0f) + 2.0f;
      }
    }
  }
}

// backward of the gate: dgate[b,h,t] -> dx_gate[b,t,h*64+c] (bf16, written densely: every head slice of every row),
// dW[o,c], db[o], d grep_a[h].   dW rows 0-3 are identical (= d wa) and rows 4-7 identical (= d wb).
// One warp per row; EIGHT lanes per head (8 columns = one 16-byte vector each), so a warp covers four heads per iteration and
// the two dot products of a head are 3-step shuffle reductions over 8 lanes (the earlier one-head-per-warp mapping spent its
// time in 5-step, 32-lane reductions: 62 us per WavLM-Large layer for 32 MB of traffic).
template <int NG>  // head groups of four per row: ceil(H / 4), all of a row's loads are issued before the first use
__global__ void __launch_bounds__(256) gate_bwd_kernel(const __nv_bfloat16* __restrict__ x, RowView xv, int H, int T,
                                                       long long rows, const float* __restrict__ grep_w,
                                                       const float* __restrict__ grep_b, const float* __restrict__ grep_a,
                                                       const float* __restrict__ dgate, __nv_bfloat16* __restrict__ dxg,
                                                       RowView dxv, float* __restrict__ dgrep_w,
                                                       float* __restrict__ dgrep_b, float* __restrict__ dgrep_a,
                                                       const int* __restrict__ valid) {
  pdl_grid_sync();
  const int lane = threadIdx.x & 31;
  const int warp = threadIdx.x >> 5;
  const int hs = lane >> 3;   // head slot inside the group of four heads
  const int q = lane & 7;     // which 8 of the head's 64 columns
  const long long warp_global = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  const long long nwarps = (static_cast<long long>(gridDim.x) * blockDim.x) >> 5;
  float wa[8], wb[8], ba = 0.f, bb = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) wa[i] = wb[i] = 0.f;
#pragma unroll
  for (int o = 0; o < 4; ++o) {
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      wa[i] += grep_w[o * 64 + q * 8 + i];
      wb[i] += grep_w[(o + 4) * 64 + q * 8 + i];
    }
    ba += grep_b[o];
    bb += grep_b[o + 4];
  }
  float dwa[8], dwb[8], dba = 0.f, dbb = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) dwa[i] = dwb[i] = 0.f;
  extern __shared__ float dga_smem[];  // [warps][H] partial d grep_a
  for (int h = lane; h < H; h += 32) dga_smem[warp * H + h] = 0.f;
  __syncwarp();
  for (long long r = warp_global; r < rows; r += nwarps) {
    const __nv_bfloat16* xr = x + xv.off(r);
    __nv_bfloat16* dr = dxg + dxv.off(r);
    const unsigned ub = static_cast<unsigned>(r) / static_cast<unsigned>(T);
    const long long b = ub, t = static_cast<unsigned>(r) - ub * static_cast<unsigned>(T);
    if (valid != nullptr && t >= valid[b]) {  // ragged batch: padded frame, zero gradient row, nothing read
#pragma unroll
      for (int gi = 0; gi < NG; ++gi) {
        const int h = gi * 4 + hs;
        if (h < H) *reinterpret_cast<uint4*>(dr + h * 64 + q * 8) = make_uint4(0u, 0u, 0u, 0u);
      }
      continue;
    }
    uint4 raw[NG];
    float dgs[NG], as[NG];
#pragma unroll
    for (int gi = 0; gi < NG; ++gi) {
      const int h = gi * 4 + hs;
      const bool live = h < H;
      raw[gi] = live ? *reinterpret_cast<const uint4*>(xr + h * 64 + q * 8) : make_uint4(0u, 0u, 0u, 0u);
      dgs[gi] = live ? dgate[(b * H + h) * T + t] : 0.f;
      as[gi] = live ? grep_a[h] : 0.f;
    }
#pragma unroll
    for (int gi = 0; gi < NG; ++gi) {
      const int h = gi * 4 + hs;
      const bool live = h < H;
      float f[8];
      {
        const uint32_t u[4] = {raw[gi].x, raw[gi].y, raw[gi].z, raw[gi].w};
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const float2 t2 = unpack_bf16x2(u[k]);
          f[2 * k] = t2.x;
          f[2 * k + 1] = t2.y;
        }
      }
      const float dg = dgs[gi];
      const float a = as[gi];
      float pa = 0.f, pb = 0.f;
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        pa = fmaf(f[i], wa[i], pa);
        pb = fmaf(f[i], wb[i], pb);
      }
#pragma unroll
      for (int o = 1; o < 8; o <<= 1) {  // the 8 lanes of a head are contiguous: xor 1, 2, 4 stays inside the group
        pa += __shfl_xor_sync(0xffffffffu, pa, o);
        pb += __shfl_xor_sync(0xffffffffu, pb, o);
      }
      const float ga = 1.0f / (1.0f + __expf(-(pa + ba)));
      const float gb = 1.0f / (1.0f + __expf(-(pb + bb)));
      const float dsa = dg * (gb * a - 1.0f) * ga * (1.0f - ga);
      const float dsb = dg * ga * a * gb * (1.0f - gb);
      float o8[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        dwa[i] = fmaf(dsa, f[i], dwa[i]);
        dwb[i] = fmaf(dsb, f[i], dwb[i]);
        o8[i] = dsa * wa[i] + dsb * wb[i];
      }
      if (live) {
        if (q == 0) {
          dba += dsa;
          dbb += dsb;
          dga_smem[warp * H + h] += dg * ga * gb;
        }
        VecIO<8>::store(dr + h * 64 + q * 8, o8);
      }
    }
  }
  // block-level reduction first (one set of global atomics per block, not per warp: all blocks hit the same 1 KB):
  // column c of d wa / d wb is spread over the 4 head slots of every warp
  __shared__ float red_w[8][4][130];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    red_w[warp][hs][q * 8 + i] = dwa[i];
    red_w[warp][hs][64 + q * 8 + i] = dwb[i];
  }
  if (q == 0) {
    red_w[warp][hs][128] = dba;
    red_w[warp][hs][129] = dbb;
  }
  __syncthreads();
  const int nw = blockDim.x >> 5;
  if (threadIdx.x < 130) {
    float s = 0.f;
    for (int w8 = 0; w8 < nw; ++w8)
#pragma unroll
      for (int k = 0; k < 4; ++k) s += red_w[w8][k][threadIdx.x];
    // every one of the 4 rows that were summed receives the same gradient
    if (threadIdx.x < 128) {
      const int half = threadIdx.x >> 6, c = threadIdx.x & 63;
#pragma unroll
      for (int o = 0; o < 4; ++o) atomicAdd(dgrep_w + (o + 4 * half) * 64 + c, s);
    } else {
      const int half = threadIdx.x - 128;
#pragma unroll
      for (int o = 0; o < 4; ++o) atomicAdd(dgrep_b + o + 4 * half, s);
    }
  }
  for (int h = threadIdx.x; h < H; h += blockDim.x) {
    float s = 0.f;
    for (int w8 = 0; w8 < nw; ++w8) s += dga_smem[w8 * H + h];
    atomicAdd(dgrep_a + h, s);
  }
}

// ------------------------------------------------------------------------------------------------ relative position table
// tab[h, i] = E[lut[i], h], i = delta + T - 1  (Toeplitz form of compute_bias, WavLM/modules.py:445-455; SURVEY.md S7)
__global__ void relpos_table_fwd_kernel(const float* __restrict__ emb, const int* __restrict__ lut, int n, int H,
                                        float* __restrict__ tab) {
  pdl_grid_sync();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n * H) return;
  const int h = i / n, d = i % n;
  tab[i] = emb[lut[d] * H + h];
}
__global__ void relpos_table_bwd_kernel(const float* __restrict__ dtab, const int* __restrict__ lut, int n, int H,
                                        float* __restrict__ demb) {
  pdl_grid_sync();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n * H) return;
  const int h = i / n, d = i % n;
  atomicAdd(demb + lut[d] * H + h, dtab[i]);
}

}  // namespace b200

using namespace b200;

extern "C" {

}  // extern "C"

static int layer_norm_fwd_impl(const void* x, long long x_bs, long long x_rs, const float* gamma, const float* beta, void* y,
                               long long y_bs, long long y_rs, float* mean, float* rstd, int rows_per_batch, int batches,
                               int D, int gelu, const int* valid, b200s_stream stream) {
  B200_CHECK_ARG(x && gamma && beta && y, "layer_norm_fwd: null pointer");
  const long long rows = static_cast<long long>(rows_per_batch) * batches;
  if (rows == 0) return 0;
  RowView xv{x_bs, x_rs, rows_per_batch}, yv{y_bs, y_rs, rows_per_batch};
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const GateArgs no_gate{nullptr, nullptr, nullptr, nullptr, 0, 1};
  int rc = dispatch_width(D, [&](auto vec, auto nch) {
    if (gelu) {
      B200_CHECK_CUDA(launch_pdl(ln_fwd_kernel<decltype(vec)::value, decltype(nch)::value, false, true>, dim3(ln_fwd_grid(rows)),
                                 dim3(256), 0, st, static_cast<const __nv_bfloat16*>(x), xv, gamma, beta,
                                 static_cast<__nv_bfloat16*>(y), yv, mean, rstd, rows, 1e-5f, no_gate, valid));
    } else {
      B200_CHECK_CUDA(launch_pdl(ln_fwd_kernel<decltype(vec)::value, decltype(nch)::value, false, false>, dim3(ln_fwd_grid(rows)),
                                 dim3(256), 0, st, static_cast<const __nv_bfloat16*>(x), xv, gamma, beta,
                                 static_cast<__nv_bfloat16*>(y), yv, mean, rstd, rows, 1e-5f, no_gate, valid));
    }
    return 0;
  });
  if (rc) return rc;
  B200_CHECK_LAUNCH();
  return 0;
}

// LayerNorm forward that also writes the gru_rel_pos gate of the attention consuming y (replaces b200s_gate_fwd + one pass
// over y).  D = H * 64 in {256, 512, 768, 1024}; x/y contiguous-row views as in b200s_layer_norm_fwd; gate: fp32 [B, H, T].
// At 512 / 768 / 1024 this is the one LayerNorm that runs the block-per-row-group kernel; every other LayerNorm call uses the
// warp-per-row kernels at all widths -- one block barrier per row group stalls all of a block's warps on the same loads, while
// independent warp-per-row chains overlap better.
static int layer_norm_gate_fwd_impl(const void* x, long long x_bs, long long x_rs, const float* gamma, const float* beta, void* y,
                                    long long y_bs, long long y_rs, float* mean, float* rstd, int T, int B, int D,
                                    const float* grep_w, const float* grep_b, const float* grep_a, int H, float* gate,
                                    const int* valid, b200s_stream stream) {
  B200_CHECK_ARG(x && gamma && beta && y && grep_w && grep_b && grep_a && gate, "layer_norm_gate_fwd: null pointer");
  B200_CHECK_ARG(D == H * 64 && (D == 256 || D == 512 || D == 768 || D == 1024),
                 "layer_norm_gate_fwd: D=%d must be H*64 and one of 256/512/768/1024", D);
  const long long rows = static_cast<long long>(T) * B;
  if (rows == 0) return 0;
  RowView xv{x_bs, x_rs, T}, yv{y_bs, y_rs, T};
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const GateArgs ga{grep_w, grep_b, grep_a, gate, H, T};
  if (D != 256) {
    return launch_ln_fwd_wide(D, rows, st, static_cast<const __nv_bfloat16*>(x), xv, gamma, beta, static_cast<__nv_bfloat16*>(y),
                              yv, mean, rstd, rows, 1e-5f, ga, valid);
  }
  B200_CHECK_CUDA(launch_pdl(ln_fwd_kernel<8, 1, true, false>, dim3(ln_fwd_grid(rows)), dim3(256), 0, st,
                             static_cast<const __nv_bfloat16*>(x), xv, gamma, beta, static_cast<__nv_bfloat16*>(y), yv, mean, rstd,
                             rows, 1e-5f, ga, valid));
  B200_CHECK_LAUNCH();
  return 0;
}

static int layer_norm_bwd_impl(const void* dy, long long dy_bs, long long dy_rs, const void* x, long long x_bs, long long x_rs,
                               const float* mean, const float* rstd, const float* gamma, const float* beta, const void* dres,
                               long long dres_bs, long long dres_rs, void* dx, long long dx_bs, long long dx_rs, float* dgamma,
                               float* dbeta, float* colsum, int rows_per_batch, int batches, int D, int gelu,
                               const int* valid, b200s_stream stream) {
  B200_CHECK_ARG(dy && x && mean && rstd && gamma && dx, "layer_norm_bwd: null pointer");
  B200_CHECK_ARG(!gelu || beta, "layer_norm_bwd: gelu mode needs beta");
  const long long rows = static_cast<long long>(rows_per_batch) * batches;
  if (rows == 0) return 0;
  RowView dyv{dy_bs, dy_rs, rows_per_batch}, xv{x_bs, x_rs, rows_per_batch}, rv{dres_bs, dres_rs, rows_per_batch},
      dxv{dx_bs, dx_rs, rows_per_batch};
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  long long blocks = ceil_div_ll(rows, 8 * 4);  // >=4 rows per warp so the column partial sums amortise
  const long long cap = static_cast<long long>(sm_count()) * 2;
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  const size_t smem = sizeof(float) * static_cast<size_t>(3 * 8 + 2) * D;  // column partials per warp + gamma + beta
  int rc = dispatch_width(D, [&](auto vec, auto nch) {
    auto kern = ln_bwd_kernel<decltype(vec)::value, decltype(nch)::value>;
    B200_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
    B200_CHECK_CUDA(launch_pdl(kern, dim3(static_cast<int>(blocks)), dim3(256), smem, st,
                               static_cast<const __nv_bfloat16*>(dy), dyv, static_cast<const __nv_bfloat16*>(x), xv, mean, rstd,
                               gamma, beta, static_cast<const __nv_bfloat16*>(dres), rv, static_cast<__nv_bfloat16*>(dx), dxv,
                               dgamma, dbeta, colsum, rows, gelu, valid));
    return 0;
  });
  if (rc) return rc;
  B200_CHECK_LAUNCH();
  return 0;
}

static int colsum_impl(const void* x, long long x_bs, long long x_rs, int rows_per_batch, int batches, int N, float* out,
                       const int* valid, b200s_stream stream) {
  B200_CHECK_ARG(x && out, "colsum: null pointer");
  B200_CHECK_ARG(N % 8 == 0, "colsum: N must be a multiple of 8");
  const long long rows = static_cast<long long>(rows_per_batch) * batches;
  if (rows == 0) return 0;
  RowView xv{x_bs, x_rs, rows_per_batch};
  const int gx = ceil_div(N, 256);
  int gy = static_cast<int>(std::min<long long>(ceil_div_ll(rows, 32), std::max(1, 4 * sm_count() / gx)));
  dim3 grid(gx, std::max(1, gy));
  B200_CHECK_CUDA(launch_pdl(colsum_kernel, dim3(grid), dim3(256), 0, static_cast<cudaStream_t>(stream),
                             static_cast<const __nv_bfloat16*>(x), xv, N, rows, out, valid));
  B200_CHECK_LAUNCH();
  return 0;
}

extern "C" {

int b200s_layer_norm_fwd(const void* x, long long x_bs, long long x_rs, const float* gamma, const float* beta, void* y,
                         long long y_bs, long long y_rs, float* mean, float* rstd, int rows_per_batch, int batches,
                         int D, int gelu, b200s_stream stream) {
  return layer_norm_fwd_impl(x, x_bs, x_rs, gamma, beta, y, y_bs, y_rs, mean, rstd, rows_per_batch, batches, D, gelu, nullptr, stream);
}
int b200s_layer_norm_fwd_ragged(const void* x, long long x_bs, long long x_rs, const float* gamma, const float* beta, void* y,
                                long long y_bs, long long y_rs, float* mean, float* rstd, int rows_per_batch, int batches,
                                int D, int gelu, const int* valid, b200s_stream stream) {
  return layer_norm_fwd_impl(x, x_bs, x_rs, gamma, beta, y, y_bs, y_rs, mean, rstd, rows_per_batch, batches, D, gelu, valid, stream);
}
int b200s_layer_norm_gate_fwd(const void* x, long long x_bs, long long x_rs, const float* gamma, const float* beta, void* y,
                              long long y_bs, long long y_rs, float* mean, float* rstd, int T, int B, int D,
                              const float* grep_w, const float* grep_b, const float* grep_a, int H, float* gate,
                              b200s_stream stream) {
  return layer_norm_gate_fwd_impl(x, x_bs, x_rs, gamma, beta, y, y_bs, y_rs, mean, rstd, T, B, D, grep_w, grep_b, grep_a, H, gate,
                                  nullptr, stream);
}
int b200s_layer_norm_gate_fwd_ragged(const void* x, long long x_bs, long long x_rs, const float* gamma, const float* beta,
                                     void* y, long long y_bs, long long y_rs, float* mean, float* rstd, int T, int B, int D,
                                     const float* grep_w, const float* grep_b, const float* grep_a, int H, float* gate,
                                     const int* valid, b200s_stream stream) {
  return layer_norm_gate_fwd_impl(x, x_bs, x_rs, gamma, beta, y, y_bs, y_rs, mean, rstd, T, B, D, grep_w, grep_b, grep_a, H, gate,
                                  valid, stream);
}
int b200s_layer_norm_bwd(const void* dy, long long dy_bs, long long dy_rs, const void* x, long long x_bs, long long x_rs,
                         const float* mean, const float* rstd, const float* gamma, const float* beta, const void* dres,
                         long long dres_bs, long long dres_rs, void* dx, long long dx_bs, long long dx_rs, float* dgamma,
                         float* dbeta, float* colsum, int rows_per_batch, int batches, int D, int gelu,
                         b200s_stream stream) {
  return layer_norm_bwd_impl(dy, dy_bs, dy_rs, x, x_bs, x_rs, mean, rstd, gamma, beta, dres, dres_bs, dres_rs, dx, dx_bs, dx_rs,
                             dgamma, dbeta, colsum, rows_per_batch, batches, D, gelu, nullptr, stream);
}
int b200s_layer_norm_bwd_ragged(const void* dy, long long dy_bs, long long dy_rs, const void* x, long long x_bs, long long x_rs,
                                const float* mean, const float* rstd, const float* gamma, const float* beta, const void* dres,
                                long long dres_bs, long long dres_rs, void* dx, long long dx_bs, long long dx_rs, float* dgamma,
                                float* dbeta, float* colsum, int rows_per_batch, int batches, int D, int gelu,
                                const int* valid, b200s_stream stream) {
  return layer_norm_bwd_impl(dy, dy_bs, dy_rs, x, x_bs, x_rs, mean, rstd, gamma, beta, dres, dres_bs, dres_rs, dx, dx_bs, dx_rs,
                             dgamma, dbeta, colsum, rows_per_batch, batches, D, gelu, valid, stream);
}
int b200s_colsum(const void* x, long long x_bs, long long x_rs, int rows_per_batch, int batches, int N, float* out,
                 b200s_stream stream) {
  return colsum_impl(x, x_bs, x_rs, rows_per_batch, batches, N, out, nullptr, stream);
}
int b200s_colsum_ragged(const void* x, long long x_bs, long long x_rs, int rows_per_batch, int batches, int N, float* out,
                        const int* valid, b200s_stream stream) {
  return colsum_impl(x, x_bs, x_rs, rows_per_batch, batches, N, out, valid, stream);
}

int b200s_dgelu_mul_ex(const void* dy, long long dy_bs, long long dy_rs, const void* pre, long long pre_bs, long long pre_rs,
                       void* out, long long out_bs, long long out_rs, int rows_per_batch, int batches, int N, float* colsum,
                       int pre_is_grad, b200s_stream stream) {
  B200_CHECK_ARG(dy && pre && out, "dgelu_mul: null pointer");
  B200_CHECK_ARG(N % 2 == 0, "dgelu_mul: N must be even");
  const long long rows = static_cast<long long>(rows_per_batch) * batches;
  if (rows == 0) return 0;
  RowView a{dy_bs, dy_rs, rows_per_batch}, b{pre_bs, pre_rs, rows_per_batch}, c{out_bs, out_rs, rows_per_batch};
  int gy = static_cast<int>(std::min<long long>(ceil_div_ll(rows, 64), 4LL * sm_count() / std::max(1, ceil_div(N, 64)) + 1));
  dim3 grid(ceil_div(N, 64), std::max(1, gy));
  B200_CHECK_CUDA(launch_pdl(dgelu_mul_kernel, dim3(grid), dim3(256), 0, static_cast<cudaStream_t>(stream), 
      static_cast<const __nv_bfloat16*>(dy), a, static_cast<const __nv_bfloat16*>(pre), b,
      static_cast<__nv_bfloat16*>(out), c, N, rows, colsum, pre_is_grad));
  B200_CHECK_LAUNCH();
  return 0;
}

int b200s_dgelu_mul(const void* dy, long long dy_bs, long long dy_rs, const void* pre, long long pre_bs, long long pre_rs,
                    void* out, long long out_bs, long long out_rs, int rows_per_batch, int batches, int N, float* colsum,
                    b200s_stream stream) {
  return b200s_dgelu_mul_ex(dy, dy_bs, dy_rs, pre, pre_bs, pre_rs, out, out_bs, out_rs, rows_per_batch, batches, N, colsum, 0,
                            stream);
}

// host evaluation of the mask formulas of dropout.cuh (no device involved): lets CPU-only tests hold the numpy restatement used
// by the parity tests to the code the kernels compile
uint32_t b200s_dropout_bits(uint32_t key0, uint32_t key1, uint32_t ctr) { return drop_bits(key0, key1, ctr); }
uint32_t b200s_dropout_row_key(uint32_t key, uint32_t row, int which) {
  return which == 0 ? drop_row_k0(key, row) : drop_row_k1(key, row);
}
uint32_t b200s_dropout_threshold16(float p) { return drop_threshold16(p); }

int b200s_dropout_rows(const void* x, long long x_bs, long long x_rs, const void* res, long long res_bs, long long res_rs,
                       void* y, long long y_bs, long long y_rs, int rows_per_batch, int batches, int N, float p,
                       uint32_t key0, uint32_t key1, b200s_stream stream) {
  B200_CHECK_ARG(x && y, "dropout_rows: null pointer");
  B200_CHECK_ARG(N > 0 && N % 8 == 0, "dropout_rows: N=%d must be a positive multiple of 8", N);
  B200_CHECK_ARG(p >= 0.f && p < 1.f, "dropout_rows: p=%f out of range [0,1)", static_cast<double>(p));
  const long long rows = static_cast<long long>(rows_per_batch) * batches;
  if (rows == 0) return 0;
  B200_CHECK_ARG(rows * N < (1LL << 32), "dropout_rows: %lld x %d elements exceed the 32-bit mask counter", rows, N);
  RowView xv{x_bs, x_rs, rows_per_batch}, rv{res_bs, res_rs, rows_per_batch}, yv{y_bs, y_rs, rows_per_batch};
  const unsigned total = static_cast<unsigned>(rows * (N / 8));
  const int grid = static_cast<int>(std::min<long long>(ceil_div_ll(total, 256), 16LL * sm_count()));
  const uint32_t thr_hi = drop_threshold16(p) << 16;
  const float rp = 1.0f / (1.0f - p);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (res != nullptr) {
    B200_CHECK_CUDA(launch_pdl(dropout_rows_kernel<true>, dim3(grid), dim3(256), 0, st, static_cast<const __nv_bfloat16*>(x), xv,
                               static_cast<const __nv_bfloat16*>(res), rv, static_cast<__nv_bfloat16*>(y), yv, N, total, key0,
                               key1, thr_hi, rp));
  } else {
    B200_CHECK_CUDA(launch_pdl(dropout_rows_kernel<false>, dim3(grid), dim3(256), 0, st, static_cast<const __nv_bfloat16*>(x), xv,
                               static_cast<const __nv_bfloat16*>(nullptr), rv, static_cast<__nv_bfloat16*>(y), yv, N, total,
                               key0, key1, thr_hi, rp));
  }
  B200_CHECK_LAUNCH();
  return 0;
}

int b200s_sumsq_rows(const void* x, long long x_bs, long long x_rs, int rows_per_batch, int batches, int N, double* out,
                     b200s_stream stream) {
  B200_CHECK_ARG(x && out, "sumsq_rows: null pointer");
  B200_CHECK_ARG(N > 0 && N % 8 == 0, "sumsq_rows: N=%d must be a positive multiple of 8", N);
  const long long rows = static_cast<long long>(rows_per_batch) * batches;
  if (rows == 0) return 0;
  B200_CHECK_ARG(rows * (N / 8) < (1LL << 32), "sumsq_rows: too many elements");
  RowView xv{x_bs, x_rs, rows_per_batch};
  const unsigned total = static_cast<unsigned>(rows * (N / 8));
  const int grid = static_cast<int>(std::min<long long>(ceil_div_ll(total, 256), 8LL * sm_count()));
  B200_CHECK_CUDA(launch_pdl(sumsq_rows_kernel, dim3(grid), dim3(256), 0, static_cast<cudaStream_t>(stream),
                             static_cast<const __nv_bfloat16*>(x), xv, N, total, out));
  B200_CHECK_LAUNCH();
  return 0;
}

int b200s_grad_multiply(void* g, long long g_bs, long long g_rs, const void* x, long long x_bs, long long x_rs,
                        int rows_per_batch, int batches, int N, float scale, const float* pen_grad, float pen_mul,
                        b200s_stream stream) {
  B200_CHECK_ARG(g, "grad_multiply: null pointer");
  B200_CHECK_ARG(pen_grad == nullptr || x != nullptr, "grad_multiply: the penalty gradient needs the features");
  B200_CHECK_ARG(N > 0 && N % 8 == 0, "grad_multiply: N=%d must be a positive multiple of 8", N);
  const long long rows = static_cast<long long>(rows_per_batch) * batches;
  if (rows == 0) return 0;
  B200_CHECK_ARG(rows * (N / 8) < (1LL << 32), "grad_multiply: too many elements");
  RowView gv{g_bs, g_rs, rows_per_batch}, xv{x_bs, x_rs, rows_per_batch};
  const unsigned total = static_cast<unsigned>(rows * (N / 8));
  const int grid = static_cast<int>(std::min<long long>(ceil_div_ll(total, 256), 16LL * sm_count()));
  B200_CHECK_CUDA(launch_pdl(grad_multiply_kernel, dim3(grid), dim3(256), 0, static_cast<cudaStream_t>(stream),
                             static_cast<__nv_bfloat16*>(g), gv, static_cast<const __nv_bfloat16*>(x), xv, N, total, scale,
                             pen_grad, pen_mul));
  B200_CHECK_LAUNCH();
  return 0;
}

int b200s_frame_mask_fwd(void* x, long long x_bs, long long x_rs, int T, int B, int D, const uint8_t* mask,
                         const uint8_t* pad, const float* mask_emb, const uint8_t* chan_mask, b200s_stream stream) {
  B200_CHECK_ARG(x, "frame_mask_fwd: null pointer");
  B200_CHECK_ARG(D % 2 == 0, "frame_mask_fwd: D must be even");
  B200_CHECK_ARG(!mask || mask_emb, "frame_mask_fwd: mask needs mask_emb");
  if (!mask && !pad && !chan_mask) return 0;
  const long long rows = static_cast<long long>(T) * B;
  RowView xv{x_bs, x_rs, T};
  auto kern = chan_mask ? frame_mask_fwd_kernel<true> : frame_mask_fwd_kernel<false>;
  B200_CHECK_CUDA(launch_pdl(kern, dim3(row_grid(rows, 8)), dim3(256), 0, static_cast<cudaStream_t>(stream),
      static_cast<__nv_bfloat16*>(x), xv, D, rows, mask, pad, mask_emb, chan_mask));
  B200_CHECK_LAUNCH();
  return 0;
}

int b200s_frame_mask_bwd(void* dx, long long x_bs, long long x_rs, int T, int B, int D, const uint8_t* mask,
                         const uint8_t* pad, float* dmask_emb, const uint8_t* chan_mask, b200s_stream stream) {
  B200_CHECK_ARG(dx, "frame_mask_bwd: null pointer");
  B200_CHECK_ARG(D <= 2048 && D % 2 == 0, "frame_mask_bwd: D=%d must be even and <= 2048", D);
  if (!mask && !pad && !chan_mask) return 0;
  const long long rows = static_cast<long long>(T) * B;
  RowView xv{x_bs, x_rs, T};
  auto kern = chan_mask ? frame_mask_bwd_kernel<true> : frame_mask_bwd_kernel<false>;
  B200_CHECK_CUDA(launch_pdl(kern, dim3(row_grid(rows, 8)), dim3(256), 0, static_cast<cudaStream_t>(stream),
      static_cast<__nv_bfloat16*>(dx), xv, D, rows, mask, pad, dmask_emb, chan_mask));
  B200_CHECK_LAUNCH();
  return 0;
}

int b200s_gate_fwd(const void* x, long long x_bs, long long x_rs, int T, int B, int H, const float* grep_w,
                   const float* grep_b, const float* grep_a, float* gate, b200s_stream stream) {
  B200_CHECK_ARG(x && grep_w && grep_b && grep_a && gate, "gate_fwd: null pointer");
  const long long rows = static_cast<long long>(T) * B;
  RowView xv{x_bs, x_rs, T};
  B200_CHECK_CUDA(launch_pdl(gate_fwd_kernel, dim3(row_grid(rows, 8)), dim3(256), 0, static_cast<cudaStream_t>(stream), 
      static_cast<const __nv_bfloat16*>(x), xv, H, T, rows, grep_w, grep_b, grep_a, gate));
  B200_CHECK_LAUNCH();
  return 0;
}

}  // extern "C"

static int gate_bwd_impl(const void* x, long long x_bs, long long x_rs, int T, int B, int H, const float* grep_w,
                         const float* grep_b, const float* grep_a, const float* dgate, void* dxg, long long dx_bs,
                         long long dx_rs, float* dgrep_w, float* dgrep_b, float* dgrep_a, const int* valid, b200s_stream stream) {
  B200_CHECK_ARG(x && grep_w && grep_b && grep_a && dgate && dxg && dgrep_w && dgrep_b && dgrep_a,
                 "gate_bwd: null pointer");
  const long long rows = static_cast<long long>(T) * B;
  RowView xv{x_bs, x_rs, T}, dv{dx_bs, dx_rs, T};
  long long blocks = std::min<long long>(ceil_div_ll(rows, 8 * 2), 4LL * sm_count());  // (2 x SMs measured 60 % slower: the row loop is latency-bound)
  if (blocks < 1) blocks = 1;
  B200_CHECK_ARG(H >= 1 && H <= 16, "gate_bwd: H=%d heads (supported: 1..16)", H);
  auto go = [&](auto ng) {
    B200_CHECK_CUDA(launch_pdl(gate_bwd_kernel<decltype(ng)::value>, dim3(static_cast<int>(blocks)), dim3(256), 8 * H * sizeof(float),
                               static_cast<cudaStream_t>(stream), static_cast<const __nv_bfloat16*>(x), xv, H, T, rows, grep_w,
                               grep_b, grep_a, dgate, static_cast<__nv_bfloat16*>(dxg), dv, dgrep_w, dgrep_b, dgrep_a, valid));
    return 0;
  };
  const int ng = (H + 3) / 4;
  const int rcg = ng == 1 ? go(std::integral_constant<int, 1>{}) : ng == 2 ? go(std::integral_constant<int, 2>{})
                : ng == 3 ? go(std::integral_constant<int, 3>{}) : go(std::integral_constant<int, 4>{});
  if (rcg) return rcg;
  B200_CHECK_LAUNCH();
  return 0;
}

extern "C" {

int b200s_gate_bwd(const void* x, long long x_bs, long long x_rs, int T, int B, int H, const float* grep_w,
                   const float* grep_b, const float* grep_a, const float* dgate, void* dxg, long long dx_bs,
                   long long dx_rs, float* dgrep_w, float* dgrep_b, float* dgrep_a, b200s_stream stream) {
  return gate_bwd_impl(x, x_bs, x_rs, T, B, H, grep_w, grep_b, grep_a, dgate, dxg, dx_bs, dx_rs, dgrep_w, dgrep_b, dgrep_a, nullptr,
                       stream);
}
int b200s_gate_bwd_ragged(const void* x, long long x_bs, long long x_rs, int T, int B, int H, const float* grep_w,
                          const float* grep_b, const float* grep_a, const float* dgate, void* dxg, long long dx_bs,
                          long long dx_rs, float* dgrep_w, float* dgrep_b, float* dgrep_a, const int* valid,
                          b200s_stream stream) {
  return gate_bwd_impl(x, x_bs, x_rs, T, B, H, grep_w, grep_b, grep_a, dgate, dxg, dx_bs, dx_rs, dgrep_w, dgrep_b, dgrep_a, valid,
                       stream);
}

int b200s_relpos_table_fwd(const float* emb, const int* lut, int n, int H, float* tab, b200s_stream stream) {
  B200_CHECK_ARG(emb && lut && tab, "relpos_table_fwd: null pointer");
  B200_CHECK_CUDA(launch_pdl(relpos_table_fwd_kernel, dim3(ceil_div(n * H, 256)), dim3(256), 0, static_cast<cudaStream_t>(stream), emb, lut, n, H, tab));
  B200_CHECK_LAUNCH();
  return 0;
}
int b200s_relpos_table_bwd(const float* dtab, const int* lut, int n, int H, float* demb, b200s_stream stream) {
  B200_CHECK_ARG(dtab && lut && demb, "relpos_table_bwd: null pointer");
  B200_CHECK_CUDA(launch_pdl(relpos_table_bwd_kernel, dim3(ceil_div(n * H, 256)), dim3(256), 0, static_cast<cudaStream_t>(stream), dtab, lut, n, H, demb));
  B200_CHECK_LAUNCH();
  return 0;
}

}  // extern "C"

extern "C" {

// LayerNorm forward with an e4m3 output (and optionally bf16 y, statistics, the fused gate): the fp8 inference path.  The
// warp-per-row kernel at every width, gate included (D = H * 64 in 256..1280).
int b200s_layer_norm_fwd_fp8(const void* x, long long x_bs, long long x_rs, const float* gamma, const float* beta, void* y,
                             long long y_bs, long long y_rs, float* mean, float* rstd, void* q, long long q_bs, long long q_rs,
                             float* scale, int rows_per_batch, int batches, int D, const float* grep_w, const float* grep_b,
                             const float* grep_a, int H, float* gate, const int* valid, b200s_stream stream) {
  B200_CHECK_ARG(x && gamma && beta && q && scale, "layer_norm_fwd_fp8: null pointer");
  B200_CHECK_ARG(!gate || (grep_w && grep_b && grep_a), "layer_norm_fwd_fp8: the gate needs grep_w, grep_b and grep_a");
  B200_CHECK_ARG(!gate || (D == H * 64 && D >= 256 && D <= 1280), "layer_norm_fwd_fp8: the fused gate needs D = H*64 in 256..1280");
  B200_CHECK_ARG(q_rs % 8 == 0 && q_bs % 8 == 0 && (reinterpret_cast<uintptr_t>(q) & 7) == 0,
                 "layer_norm_fwd_fp8: e4m3 rows must be 8-byte aligned");
  const long long rows = static_cast<long long>(rows_per_batch) * batches;
  if (rows == 0) return 0;
  RowView xv{x_bs, x_rs, rows_per_batch}, yv{y_bs, y_rs, rows_per_batch};
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const GateArgs ga{grep_w, grep_b, grep_a, gate, H, rows_per_batch};
  const Fp8Rows f8{static_cast<uint8_t*>(q), q_bs, q_rs, scale};
  int rc = dispatch_width(D, [&](auto vec, auto nch) {
    constexpr int V = decltype(vec)::value, NC = decltype(nch)::value;
    if constexpr (V == 8) {
      if (gate) {
        B200_CHECK_CUDA(launch_pdl(ln_fwd_fp8_kernel<V, NC, true>, dim3(ln_fwd_grid(rows)), dim3(256), 0, st,
                                   static_cast<const __nv_bfloat16*>(x), xv, gamma, beta, static_cast<__nv_bfloat16*>(y), yv, mean,
                                   rstd, rows, 1e-5f, ga, f8, valid));
        return 0;
      }
    }
    B200_CHECK_CUDA(launch_pdl(ln_fwd_fp8_kernel<V, NC, false>, dim3(ln_fwd_grid(rows)), dim3(256), 0, st,
                               static_cast<const __nv_bfloat16*>(x), xv, gamma, beta, static_cast<__nv_bfloat16*>(y), yv, mean,
                               rstd, rows, 1e-5f, ga, f8, valid));
    return 0;
  });
  if (rc) return rc;
  B200_CHECK_LAUNCH();
  return 0;
}

}  // extern "C"
