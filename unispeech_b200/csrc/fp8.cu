// FP8 (e4m3) inference path of the encoder projections (QKV, out_proj, fc1, fc2): the row GEMM on e4m3 operands, the
// quantisation of bf16 rows that no LayerNorm produces (attention output, GELU output), and the preparation of the e4m3 weights
// from the fp32 masters.  Numerics (fp8.cuh): one scale per activation row, one per weight row (output channel), fp32
// accumulation, bf16 output; the scales factor out of the K sum, so the main loop is pure e4m3 wgmma and the epilogue applies
// s[row] * sw[col] before bias, GELU and residual.
#include <algorithm>
#include <mutex>

#include "../../include/unispeech_b200.h"
#include "common.h"
#include "fp8.cuh"
#include "ptx.cuh"
#include "ws_epilogue.cuh"

namespace b200 {

int make_fp8_rows_tmap(CUtensorMap* out, const void* ptr, long long K, long long rows, long long batches, long long row_stride,
                       long long batch_stride, int box_rows);

struct Fp8Tensor {
  void* p;
  long long bs;  // batch stride (elements)
  long long ld;  // row stride (elements)
};

// D[64 x 128] (+)= A[64 x 32] * B[32 x 128], e4m3 operands K-major in shared memory (the only layout fp8 wgmma takes), fp32
// accumulators; executed by all 128 threads of a warpgroup.  scale_d = 0 overwrites D.
__device__ __forceinline__ void wgmma_m64n128k32_e4m3(float* d, uint64_t desc_a, uint64_t desc_b, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k32.f32.e4m3.e4m3 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
      "%64, %65, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(desc_a), "l"(desc_b), "r"(scale_d)
      : "memory");
}

// ------------------------------------------------------------------------------- persistent 128 x 256 fp8 row GEMM
// out[b, r, n] = epilogue(s[b, r] * sw[n] * sum_k qa[b, r, k] qw[n, k]).  gemm_ws_kernel's structure (gemm.cuh) on e4m3 operands:
//   warpgroup 0    : TMA producer (one elected lane)
//   warpgroups 1-2 : consumers, 64 rows of the tile each (wgmma m64n128k32 e4m3 per n128 half, 128 fp32 sums per thread)
// A K block is 128 e4m3 = one 128-byte swizzle row, so a stage (128 x 128 B of A, 256 x 128 B of B) and the shared-memory
// descriptors (k32 step = 32 bytes) are those of the bf16 kernel; each stage carries twice the K of a bf16 stage.
// Promotion: the tensor cores' e4m3 accumulation does not keep full fp32 precision (measured: up to 6.4e-3 of max|out| at
// K = 7680 with one accumulator over the whole K loop, against the GEMM test's bound of 4e-3; DESIGN.md section 5e).  So every
// K block (128) of each n128 half of a consumer's 64 x 256 sub-tile goes into a fresh 64-register wgmma accumulator, which is
// then added into the 128 fp32 registers of the sub-tile: 192 accumulator registers, where two full 64 x 256 copies would not fit.
// Ragged batches are handled in the persistent walk: a tile at or past valid[b] is skipped by the producer and written as zeros
// by the consumers.
struct Fp8GemmParams {
  int m_rows;             // rows per batch
  int m_tiles_per_batch;  // ceil(m_rows / 128)
  int m_tiles;            // over all batches
  int n_total;
  int k_blocks;           // K / 128
  int gelu;
  const float* a_scale;   // [batches * m_rows]
  const float* w_scale;   // [n_total]
  const float* bias;      // [n_total] or null
  Fp8Tensor out, res1;    // bf16
  const int* m_valid;     // [batches] or null
};

struct Fp8WsCfg {
  static constexpr int kStages = 3;
  static constexpr int kABytes = 128 * 128;  // 128 rows x 128 e4m3
  static constexpr int kBBytes = 256 * 128;  // 256 rows x 128 e4m3
  static constexpr int kStageBytes = kABytes + kBBytes;
  static constexpr int kEpiBytes = 64 * 64 * 4;     // one consumer warpgroup's 64 x 64 fp32 staging chunk
  static constexpr int kPfBytes = 8 * 128 * 8;      // one consumer warpgroup's prefetched residual: 8 rows x 128 threads x 4 bf16
  static constexpr int kSmemBytes = kStages * kStageBytes + 2 * kEpiBytes + 2 * kPfBytes + 1024;
  static constexpr int kThreads = 384;
  static_assert(kSmemBytes + 1024 <= 232448, "one CTA per SM");
};

__global__ void __launch_bounds__(384, 1) gemm_fp8_kernel(const __grid_constant__ CUtensorMap tmA,
                                                          const __grid_constant__ CUtensorMap tmB,
                                                          const __grid_constant__ Fp8GemmParams p) {
  pdl_launch_dependents();
  using Cfg = Fp8WsCfg;
  constexpr int kStages = Cfg::kStages;
  const int wg = threadIdx.x >> 7;
  const int lane = threadIdx.x & 31;
  const int n_tiles = (p.n_total + 255) / 256;
  const int num_tiles = p.m_tiles * n_tiles;

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  __shared__ uint64_t full_bar[kStages];
  __shared__ uint64_t empty_bar[kStages];

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
#pragma unroll
    for (int s = 0; s < kStages; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 8);  // one arrival per consumer warp
    }
    fence_mbar_init();
  }
  __syncthreads();
  pdl_wait();
  auto dead = [&](int mb, int m0) { return p.m_valid != nullptr && m0 >= __ldg(p.m_valid + mb); };

  if (wg == 0) {
    // ------------------------------------------------------------ TMA producer
    setmaxnreg_dec<40>();
    if (threadIdx.x == 0) {
      int it = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const int mt = tile / n_tiles, n_tile = tile - mt * n_tiles;
        const int mb = mt / p.m_tiles_per_batch, m0 = (mt - mb * p.m_tiles_per_batch) * 128;
        if (dead(mb, m0)) continue;
        for (int kb = 0; kb < p.k_blocks; ++kb, ++it) {
          const int s = it % kStages;
          mbar_wait(&empty_bar[s], ((it / kStages) & 1) ^ 1);
          uint8_t* sa = smem + s * Cfg::kStageBytes;
          mbar_expect_tx(&full_bar[s], Cfg::kStageBytes);
          tma_load_4d(sa, &tmA, &full_bar[s], kb * 128, m0, mb, 0);
          tma_load_4d(sa + Cfg::kABytes, &tmB, &full_bar[s], kb * 128, n_tile * 256, 0, 0);
        }
      }
    }
    return;
  }

  // -------------------------------------------------------------- consumers: warpgroup c owns rows 64 c .. 64 c + 63
  setmaxnreg_inc<232>();
  const int c = wg - 1;
  const int t = threadIdx.x & 127, w = t >> 5;
  float* stage = reinterpret_cast<float*>(smem + kStages * Cfg::kStageBytes + c * Cfg::kEpiBytes);
  uint2* pf = reinterpret_cast<uint2*>(smem + kStages * Cfg::kStageBytes + 2 * Cfg::kEpiBytes + c * Cfg::kPfBytes);
  const int cq = ws_lane_col(lane);  // epilogue: this lane's 4 columns of a 64-column chunk
  float acc[128];                  // fp32 sums of the 64 x 256 sub-tile (promoted from `part` every K block)
  float part[64];                  // one n128 half of one K block: the wgmma accumulators
  int it = 0;
  for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
    const int mt = tile / n_tiles, n_tile = tile - mt * n_tiles;
    const int mb = mt / p.m_tiles_per_batch, m0 = (mt - mb * p.m_tiles_per_batch) * 128;
    const int col_base = n_tile * 256;
    const int n_valid = min(256, p.n_total - col_base);
    const int rows_here = min(128, p.m_rows - m0) - 64 * c;  // valid rows of this warpgroup's half (may be <= 0)
    const long long row0 = static_cast<long long>(m0) + 64 * c;
    __nv_bfloat16* out = static_cast<__nv_bfloat16*>(p.out.p) + mb * p.out.bs + row0 * p.out.ld + col_base;
    if (dead(mb, m0)) {  // padded frames only: zeros (finite), nothing loaded
      for (int j = 0; j < 4; ++j) {
        const int cl = 64 * j + cq;
        if (cl >= n_valid) break;
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const int r = ws_chunk_row(w, i, lane);
          if (r < rows_here) *reinterpret_cast<uint2*>(out + r * p.out.ld + cl) = make_uint2(0u, 0u);
        }
      }
      continue;
    }
    // the 4 columns x 8 rows of chunk j's residual that this thread reads are copied into its own slots pf[i, t]
    auto prefetch = [&](int j) {
      const int cl = 64 * j + cq;
      if (p.res1.p != nullptr && cl < n_valid) {
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const int r = ws_chunk_row(w, i, lane);
          if (r < rows_here)
            cp_async_8(pf + i * 128 + t, static_cast<const __nv_bfloat16*>(p.res1.p) + mb * p.res1.bs + (row0 + r) * p.res1.ld +
                                             col_base + cl);
        }
      }
      cp_async_commit();
    };
    prefetch(0);
    float sr[8];  // row scales of this thread's 8 epilogue rows
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int r = ws_chunk_row(w, i, lane);
      sr[i] = r < rows_here ? __ldg(p.a_scale + static_cast<long long>(mb) * p.m_rows + row0 + r) : 0.f;
    }
#pragma unroll
    for (int i = 0; i < 128; ++i) acc[i] = 0.f;
    for (int kb = 0; kb < p.k_blocks; ++kb, ++it) {
      const int s = it % kStages;
      mbar_wait(&full_bar[s], (it / kStages) & 1);
      const uint32_t sa = smem_u32(smem + s * Cfg::kStageBytes) + c * 8192;  // rows 64 c .. of A: 64 rows x 128 B
      const uint32_t sb = smem_u32(smem + s * Cfg::kStageBytes + Cfg::kABytes);
#pragma unroll
      for (int h = 0; h < 2; ++h) {  // columns 128 h .. 128 h + 127 = B rows from 16 KB in (the n256 fragment's registers 64 h ..)
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < 4; ++k)
          wgmma_m64n128k32_e4m3(part, make_smem_desc_sw128(sa + k * 32, 16, 1024),
                                make_smem_desc_sw128(sb + h * 16384 + k * 32, 16, 1024), k > 0 ? 1u : 0u);
        wgmma_commit();
        wgmma_wait<0>();
#pragma unroll
        for (int i = 0; i < 64; ++i) acc[64 * h + i] += part[i];
      }
      if (lane == 0) mbar_arrive(&empty_bar[s]);  // the K block's MMAs have retired: its stage goes back to the producer
    }

    // ---- epilogue, 64 columns at a time (ws_stage_chunk): scales, bias, GELU, residual
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      if (64 * j >= n_valid) break;  // warpgroup-uniform
      named_bar_sync(1 + c, 128);    // the previous chunk has been read out of the staging buffer
      ws_stage_chunk(acc, stage, j, w, lane);
      const int cl = 64 * j + cq;
      const bool col_ok = cl < n_valid;
      named_bar_sync(1 + c, 128);
      float4 b4 = make_float4(0.f, 0.f, 0.f, 0.f), s4 = b4;
      if (col_ok) {
        s4 = __ldg(reinterpret_cast<const float4*>(p.w_scale + col_base + cl));
        if (p.bias != nullptr) b4 = __ldg(reinterpret_cast<const float4*>(p.bias + col_base + cl));
      }
      cp_async_wait_all();  // this thread's residual of chunk j has landed
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const int r = ws_chunk_row(w, i, lane);
        const float4 v4 = ws_load_row(stage, r, cq);
        if (!col_ok || r >= rows_here) continue;
        float v[4] = {v4.x * sr[i] * s4.x + b4.x, v4.y * sr[i] * s4.y + b4.y, v4.z * sr[i] * s4.z + b4.z,
                      v4.w * sr[i] * s4.w + b4.w};
        if (p.gelu) {
#pragma unroll
          for (int k = 0; k < 4; ++k) v[k] = gelu_f(v[k]);
        }
        if (p.res1.p != nullptr) add_bf16x4(v, pf[i * 128 + t]);
        *reinterpret_cast<uint2*>(out + r * p.out.ld + cl) = pack_bf16x4(v);
      }
      if (j < 3) prefetch(j + 1);  // this thread's slots have been read
    }
  }
}

// ------------------------------------------------------------------------------- bf16 rows -> e4m3 rows + row scales
// One warp per row, the row held in registers (NV 8-element vectors per lane: D <= 256 NV), so x is read once.  NV is the
// smallest of 4 / 8 / 16 / 32 that holds the row: registers, and so resident warps, follow the width.
constexpr int kQuantVecs = 32;
template <int NV>
__global__ void __launch_bounds__(256) quantize_rows_fp8_kernel(const __nv_bfloat16* __restrict__ x, long long x_bs, long long x_rs,
                                                                int rows, long long total, int D, uint8_t* __restrict__ q,
                                                                long long q_bs, long long q_rs, float* __restrict__ scale,
                                                                const int* __restrict__ valid) {
  pdl_grid_sync();
  const int lane = threadIdx.x & 31;
  const long long warp_global = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  const long long nwarps = (static_cast<long long>(gridDim.x) * blockDim.x) >> 5;
  const int nv = D / 8;
  for (long long r = warp_global; r < total; r += nwarps) {
    const long long b = r / rows, tr = r - b * rows;
    uint8_t* qr = q + b * q_bs + tr * q_rs;
    if (valid != nullptr && tr >= __ldg(valid + b)) {  // padding: zeros, s = 0, nothing read
      for (int i = lane; i < nv; i += 32) *reinterpret_cast<uint2*>(qr + 8 * i) = make_uint2(0u, 0u);
      if (lane == 0) scale[r] = 0.f;
      continue;
    }
    const __nv_bfloat16* xr = x + b * x_bs + tr * x_rs;
    uint4 raw[NV];
    float amax = 0.f;
#pragma unroll
    for (int j = 0; j < NV; ++j) {
      const int i = j * 32 + lane;
      if (i < nv) {
        raw[j] = *reinterpret_cast<const uint4*>(xr + 8 * i);
        const uint32_t u[4] = {raw[j].x, raw[j].y, raw[j].z, raw[j].w};
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const float2 f = unpack_bf16x2(u[k]);
          amax = fmaxf(amax, fmaxf(fabsf(f.x), fabsf(f.y)));
        }
      }
    }
    amax = warp_max(amax);
    const float rinv = fp8_row_rinv(amax);
#pragma unroll
    for (int j = 0; j < NV; ++j) {
      const int i = j * 32 + lane;
      if (i < nv) {
        const uint32_t u[4] = {raw[j].x, raw[j].y, raw[j].z, raw[j].w};
        float v[8];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const float2 f = unpack_bf16x2(u[k]);
          v[2 * k] = f.x;
          v[2 * k + 1] = f.y;
        }
        *reinterpret_cast<uint2*>(qr + 8 * i) = make_uint2(fp8x4(v, rinv), fp8x4(v + 4, rinv));
      }
    }
    if (lane == 0) scale[r] = fp8_row_scale(amax);
  }
}

// ------------------------------------------------------------------------------- fp32 masters -> e4m3 weights + channel scales
// One launch for every projection of the encoder (descriptor table in device memory, built once; the masters never move).
// Block (x, d): rows 8 x .. 8 x + 7 of descriptor d, one warp per row; two passes over the fp32 row (amax, then quantise).
struct Fp8PrepDesc {
  const float* src;  // [N, K] fp32
  uint8_t* dst;      // [N, K] e4m3
  float* scale;      // [N]
  int N, K;          // K % 8 == 0
};
__global__ void __launch_bounds__(256) prep_linear_fp8_batched_kernel(const Fp8PrepDesc* __restrict__ descs) {
  pdl_grid_sync();
  const Fp8PrepDesc d = descs[blockIdx.y];
  const int row = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (row >= d.N) return;
  const float* src = d.src + static_cast<long long>(row) * d.K;
  float amax = 0.f;
  for (int k = 4 * lane; k < d.K; k += 128) {
    const float4 v = *reinterpret_cast<const float4*>(src + k);
    amax = fmaxf(amax, fmaxf(fmaxf(fabsf(v.x), fabsf(v.y)), fmaxf(fabsf(v.z), fabsf(v.w))));
  }
  amax = warp_max(amax);
  const float rinv = fp8_row_rinv(amax);
  uint8_t* dst = d.dst + static_cast<long long>(row) * d.K;
  for (int k = 8 * lane; k < d.K; k += 256) {
    const float4 a = *reinterpret_cast<const float4*>(src + k), b = *reinterpret_cast<const float4*>(src + k + 4);
    const float v[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
    *reinterpret_cast<uint2*>(dst + k) = make_uint2(fp8x4(v, rinv), fp8x4(v + 4, rinv));
  }
  if (lane == 0) d.scale[row] = fp8_row_scale(amax);
}

}  // namespace b200

using namespace b200;

extern "C" {

int b200s_gemm_rows_fp8(const void* a8, const float* a_scale, long long a_bs, long long a_rs, int rows, int batches, int K,
                        const void* w8, const float* w_scale, int N, void* out, long long out_bs, long long out_ld,
                        const b200s_epilogue* epi, const int* valid, b200s_stream stream) {
  B200_CHECK_ARG(a8 && a_scale && w8 && w_scale && out, "gemm_rows_fp8: null pointer");
  B200_CHECK_ARG(rows > 0 && batches > 0 && K > 0 && N > 0, "gemm_rows_fp8: bad sizes");
  B200_CHECK_ARG(K % 128 == 0, "gemm_rows_fp8: K=%d must be a multiple of 128", K);
  B200_CHECK_ARG(N % 8 == 0, "gemm_rows_fp8: N=%d must be a multiple of 8", N);
  B200_CHECK_ARG(out_ld % 8 == 0 && (batches == 1 || out_bs % 8 == 0) && (reinterpret_cast<uintptr_t>(out) & 15) == 0,
                 "gemm_rows_fp8: output rows must be 16-byte aligned");
  if (epi) {
    B200_CHECK_ARG(!epi->res2 && !epi->gelu_aux && !epi->dgelu && !epi->out_pre && !epi->colsum,
                   "gemm_rows_fp8: the epilogue takes bias, gelu and res1 only");
    B200_CHECK_ARG(!epi->res1 || (epi->res1_ld % 8 == 0 && (batches == 1 || epi->res1_bs % 8 == 0) &&
                                  (reinterpret_cast<uintptr_t>(epi->res1) & 15) == 0),
                   "gemm_rows_fp8: residual rows must be 16-byte aligned");
    B200_CHECK_ARG(!epi->bias || (reinterpret_cast<uintptr_t>(epi->bias) & 15) == 0, "gemm_rows_fp8: bias must be 16-byte aligned");
  }
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  CUtensorMap ta, tb;
  if (make_fp8_rows_tmap(&ta, a8, K, rows, batches, a_rs, a_bs, 128)) return -3;
  if (make_fp8_rows_tmap(&tb, w8, K, N, 1, K, 0, 256)) return -3;
  Fp8GemmParams p;
  memset(&p, 0, sizeof(p));
  p.m_rows = rows;
  p.m_tiles_per_batch = ceil_div(rows, 128);
  p.m_tiles = p.m_tiles_per_batch * batches;
  p.n_total = N;
  p.k_blocks = K / 128;
  p.a_scale = a_scale;
  p.w_scale = w_scale;
  p.out = {out, out_bs, out_ld};
  p.res1 = {nullptr, 0, 0};
  p.m_valid = valid;
  if (epi) {
    p.bias = epi->bias;
    p.gelu = epi->gelu != 0;
    p.res1 = {const_cast<void*>(epi->res1), epi->res1_bs, epi->res1_ld};
  }
  static std::once_flag once;
  static cudaError_t attr_err = cudaSuccess;
  std::call_once(once, [] {
    attr_err = cudaFuncSetAttribute(gemm_fp8_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, Fp8WsCfg::kSmemBytes);
  });
  B200_CHECK_CUDA(attr_err);
  const int tiles = p.m_tiles * ceil_div(N, 256);
  B200_CHECK_CUDA(launch_pdl(gemm_fp8_kernel, dim3(std::min(tiles, sm_count())), dim3(Fp8WsCfg::kThreads), Fp8WsCfg::kSmemBytes,
                             st, ta, tb, p));
  B200_CHECK_LAUNCH();
  return 0;
}

int b200s_quantize_rows_fp8(const void* x, long long x_bs, long long x_rs, int rows, int batches, int D, void* q, long long q_bs,
                            long long q_rs, float* scale, const int* valid, b200s_stream stream) {
  B200_CHECK_ARG(x && q && scale, "quantize_rows_fp8: null pointer");
  B200_CHECK_ARG(rows >= 0 && batches >= 0, "quantize_rows_fp8: bad sizes");
  B200_CHECK_ARG(D > 0 && D % 8 == 0 && D <= 8 * 32 * kQuantVecs, "quantize_rows_fp8: D=%d must be a multiple of 8 and <= %d", D,
                 8 * 32 * kQuantVecs);
  B200_CHECK_ARG(x_rs % 8 == 0 && x_bs % 8 == 0 && q_rs % 8 == 0 && q_bs % 8 == 0 && (reinterpret_cast<uintptr_t>(x) & 15) == 0 &&
                     (reinterpret_cast<uintptr_t>(q) & 7) == 0,
                 "quantize_rows_fp8: rows must be 16-byte (x) / 8-byte (q) aligned");
  const long long total = static_cast<long long>(rows) * batches;
  if (total == 0) return 0;
  const long long blocks = std::min<long long>(ceil_div_ll(total, 8), static_cast<long long>(sm_count()) * 8);
  const int nv = ceil_div(D / 8, 32);
  auto kern = nv <= 4 ? quantize_rows_fp8_kernel<4> : nv <= 8 ? quantize_rows_fp8_kernel<8>
            : nv <= 16 ? quantize_rows_fp8_kernel<16> : quantize_rows_fp8_kernel<kQuantVecs>;
  B200_CHECK_CUDA(launch_pdl(kern, dim3(static_cast<int>(blocks)), dim3(256), 0, static_cast<cudaStream_t>(stream),
                             static_cast<const __nv_bfloat16*>(x), x_bs, x_rs, rows, total, D, static_cast<uint8_t*>(q), q_bs, q_rs,
                             scale, valid));
  B200_CHECK_LAUNCH();
  return 0;
}

int b200s_prep_linear_fp8_batched(const void* descs, int n_descs, int max_rows, b200s_stream stream) {
  B200_CHECK_ARG(descs && n_descs > 0 && n_descs <= 65535 && max_rows > 0, "prep_linear_fp8_batched: bad arguments");
  B200_CHECK_CUDA(launch_pdl(prep_linear_fp8_batched_kernel, dim3(ceil_div(max_rows, 8), n_descs), dim3(256), 0,
                             static_cast<cudaStream_t>(stream), static_cast<const Fp8PrepDesc*>(descs)));
  B200_CHECK_LAUNCH();
  return 0;
}

}  // extern "C"
