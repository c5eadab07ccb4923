// Parameter preparation kernels: fp32 master parameters in the REFERENCE state_dict layout -> bf16 operands in the layouts
// the GEMM kernels consume (and the inverse mapping for the fp32 gradients).  All tiny compared with the activations.
//   * nn.Linear  [N,K]            -> bf16 [N,K] (+ optional row scale, e.g. q * head_dim^-0.5) and its transpose [K,N]
//   * nn.Conv1d  [Co,Ci,k]        -> forward B operand [Co, k*Ci] (tap-major), per-phase input-gradient operands
//   * pos_conv   weight_norm(dim=2) [D, D/G, taps] (WavLM/WavLM.py:514-527; SURVEY.md S3) -> zero-padded per-group
//                operands for the forward and the flipped/transposed input-gradient implicit GEMMs; backward of the
//                weight normalisation.
#include "../../include/unispeech_b200.h"
#include "common.h"
#include "ptx.cuh"

namespace b200 {

__global__ void scale_copy_f32_kernel(const float* __restrict__ src, float* __restrict__ dst, long long n, float scale) {
  pdl_grid_sync();
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i < n) dst[i] = src[i] * scale;
}

// dst[n*ld + k] = bf16(src[n,k]*scale);  dstT[k*ldT + n] = same, through a 32x32 shared tile
__global__ void prep_linear_kernel(const float* __restrict__ src, int N, int K, float scale, __nv_bfloat16* __restrict__ dst,
                                   long long ld, __nv_bfloat16* __restrict__ dstT, long long ldT) {
  pdl_grid_sync();
  __shared__ float tile[32][33];
  const int n0 = blockIdx.y * 32, k0 = blockIdx.x * 32;
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int n = n0 + i, k = k0 + threadIdx.x;
    float v = 0.f;
    if (n < N && k < K) {
      v = src[static_cast<long long>(n) * K + k] * scale;
      if (dst) dst[static_cast<long long>(n) * ld + k] = __float2bfloat16_rn(v);
    }
    tile[i][threadIdx.x] = v;
  }
  __syncthreads();
  if (dstT) {
    for (int i = threadIdx.y; i < 32; i += blockDim.y) {
      const int k = k0 + i, n = n0 + threadIdx.x;
      if (n < N && k < K) dstT[static_cast<long long>(k) * ldT + n] = __float2bfloat16_rn(tile[threadIdx.x][i]);
    }
  }
}

// Batched variant: ONE launch prepares every nn.Linear operand of the model (descriptor table in device memory, built once;
// the master parameters never move).  Block -> (descriptor, 64x64 tile) by binary search over the tile prefix sums.
// The kernel is pure HBM traffic (4 B read + 2 x 2 B written per weight, 1.26 GB + 1.26 GB per WavLM-Large step): 16-byte
// loads of the fp32 rows, 8-byte stores of the bf16 rows, 128-byte rows of the transposed copy through a padded smem tile.
struct PrepLinearDesc {
  const float* src;
  __nv_bfloat16* dst;
  __nv_bfloat16* dstT;
  long long ld, ldT;
  int N, K;
  int tile_begin;  // first global tile index of this descriptor
  int tiles_k;     // ceil(K / 64)
};
constexpr int kPrepTile = 64;
__global__ void __launch_bounds__(256) prep_linear_batched_kernel(const PrepLinearDesc* __restrict__ descs, int n_descs) {
  pdl_grid_sync();
  __shared__ float tile[kPrepTile][kPrepTile + 1];
  int lo = 0, hi = n_descs - 1;
  const int t = blockIdx.x;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (descs[mid].tile_begin <= t) lo = mid; else hi = mid - 1;
  }
  const PrepLinearDesc d = descs[lo];
  const int lt = t - d.tile_begin;
  const int n0 = (lt / d.tiles_k) * kPrepTile, k0 = (lt % d.tiles_k) * kPrepTile;
  const int tid = threadIdx.x;
  {
    const int tx = tid & 15, ty = tid >> 4;  // 16 threads x 4 floats per row, 16 rows per step
    const int k = k0 + tx * 4;
    const bool vec_ok = (k + 3 < d.K) && ((d.K & 3) == 0) && ((d.ld & 3) == 0) &&
                        ((reinterpret_cast<uintptr_t>(d.src) & 15) == 0) && (d.dst == nullptr || (reinterpret_cast<uintptr_t>(d.dst) & 7) == 0);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int r = ty + 16 * i, n = n0 + r;
      float v[4] = {0.f, 0.f, 0.f, 0.f};
      if (n < d.N) {
        if (vec_ok) {
          const float4 f = *reinterpret_cast<const float4*>(d.src + static_cast<long long>(n) * d.K + k);
          v[0] = f.x; v[1] = f.y; v[2] = f.z; v[3] = f.w;
          if (d.dst) {
            uint2 w;
            w.x = pack_bf16x2(v[0], v[1]);
            w.y = pack_bf16x2(v[2], v[3]);
            *reinterpret_cast<uint2*>(d.dst + static_cast<long long>(n) * d.ld + k) = w;
          }
        } else {
#pragma unroll
          for (int e = 0; e < 4; ++e)
            if (k + e < d.K) {
              v[e] = d.src[static_cast<long long>(n) * d.K + k + e];
              if (d.dst) d.dst[static_cast<long long>(n) * d.ld + k + e] = __float2bfloat16_rn(v[e]);
            }
        }
      }
#pragma unroll
      for (int e = 0; e < 4; ++e) tile[r][tx * 4 + e] = v[e];
    }
  }
  __syncthreads();
  if (d.dstT) {
    const int tx = tid & 31, ty = tid >> 5;  // 32 threads x 2 columns (n) per transposed row, 8 rows (k) per step
    const int n = n0 + tx * 2;
    const bool pair_ok = (n + 1 < d.N) && ((d.ldT & 1) == 0) && ((reinterpret_cast<uintptr_t>(d.dstT) & 3) == 0);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int kk = ty + 8 * i, k = k0 + kk;
      if (k >= d.K) continue;
      const float a = tile[tx * 2][kk], b2 = tile[tx * 2 + 1][kk];
      __nv_bfloat16* o = d.dstT + static_cast<long long>(k) * d.ldT + n;
      if (pair_ok) {
        *reinterpret_cast<uint32_t*>(o) = pack_bf16x2(a, b2);
      } else {
        if (n < d.N) o[0] = __float2bfloat16_rn(a);
        if (n + 1 < d.N) o[1] = __float2bfloat16_rn(b2);
      }
    }
  }
}

// conv forward operand: dst[co, j*Ci + ci] = src[co, ci, j]
__global__ void prep_conv_fwd_kernel(const float* __restrict__ src, int Co, int Ci, int k, __nv_bfloat16* __restrict__ dst) {
  pdl_grid_sync();
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const long long n = static_cast<long long>(Co) * Ci * k;
  if (i >= n) return;
  const int ci = i % Ci;
  const int j = (i / Ci) % k;
  const int co = i / (static_cast<long long>(Ci) * k);
  dst[i] = __float2bfloat16_rn(src[(static_cast<long long>(co) * Ci + ci) * k + j]);
}
// conv input-gradient operand for phase rho (input row r = s*u + rho):  taps j = rho + s*m, m < nm.
// dst[ci, mm*Co + co] = src[co, ci, rho + s*(nm-1-mm)]     (A rows are [dY[u-(nm-1)], ..., dY[u]])
__global__ void prep_conv_dgrad_kernel(const float* __restrict__ src, int Co, int Ci, int k, int s, int rho, int nm,
                                       __nv_bfloat16* __restrict__ dst) {
  pdl_grid_sync();
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const long long n = static_cast<long long>(Ci) * nm * Co;
  if (i >= n) return;
  const int co = i % Co;
  const int mm = (i / Co) % nm;
  const int ci = i / (static_cast<long long>(Co) * nm);
  const int j = rho + s * (nm - 1 - mm);
  dst[i] = __float2bfloat16_rn(src[(static_cast<long long>(co) * Ci + ci) * k + j]);
}
// gradient back to the reference layout: dw[co, ci, j] += dwk[co, j*Ci + ci]
__global__ void unprep_conv_wgrad_kernel(const float* __restrict__ dwk, int Co, int Ci, int k, float* __restrict__ dw) {
  pdl_grid_sync();
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const long long n = static_cast<long long>(Co) * Ci * k;
  if (i >= n) return;
  const int j = i % k;
  const int ci = (i / k) % Ci;
  const int co = i / (static_cast<long long>(Ci) * k);
  dw[i] += dwk[(static_cast<long long>(co) * k + j) * Ci + ci];
}

// ---- pos_conv weight norm -----------------------------------------------------------------------------------------
// Channels per group Cg <= 128; the GEMM operands are padded to Cgp = 64 (Cg <= 64) or 128 channels per group (posconv_cgp).
__host__ __device__ __forceinline__ int posconv_cgp(int Cg) { return Cg <= 64 ? 64 : 128; }
// norm2[j] = sum_{co,ci} v[co,ci,j]^2  (and optionally dot[j] = sum dw*v for the backward; dwp is [G, Cg, taps, Cgp]).  The block partials are combined with
// fp64 atomics: their order varies from launch to launch, but an fp64 sum of a few hundred fp32 partials rounds to the same fp32
// value whatever the order (fp32 atomics did not: the weight norm, hence a few bf16 pos_conv weights, hence the whole forward pass
// differed in the last bit between two runs on the same input -- found by tests/test_graph_gpu.py).
__global__ void posconv_tap_reduce_kernel(const float* __restrict__ v, const float* __restrict__ dwp, int D, int Cg, int taps,
                                          double* __restrict__ norm2, double* __restrict__ dot) {
  pdl_grid_sync();
  // thread -> tap (coalesced over the contiguous tap axis), blocks stride over (co, ci) rows
  const int j = threadIdx.x;
  if (j >= taps) return;
  const long long rows = static_cast<long long>(D) * Cg;
  float a = 0.f, d = 0.f;
  for (long long r = blockIdx.x; r < rows; r += gridDim.x) {
    const float x = v[r * taps + j];
    a += x * x;
    if (dwp) {
      const int co = r / Cg, ci = r % Cg;  // co global channel
      const int g = co / Cg, cog = co % Cg;
      d += dwp[((static_cast<long long>(g) * Cg + cog) * taps + j) * posconv_cgp(Cg) + ci] * x;
    }
  }
  atomicAdd(norm2 + j, static_cast<double>(a));
  if (dwp) atomicAdd(dot + j, static_cast<double>(d));
}
// wp_fwd[(g*Cgp+co), j*Cgp+ci] = w[g*Cg+co, ci, j];   wp_dg[(g*Cgp+ci), j'*Cgp+co] = w[g*Cg+co, ci, taps-1-j']
// with w = gvec[j] * v / sqrt(norm2[j]); zero padding elsewhere.
__global__ void posconv_prep_kernel(const float* __restrict__ v, const float* __restrict__ gvec,
                                    const double* __restrict__ norm2, int G, int Cg, int taps,
                                    __nv_bfloat16* __restrict__ wp_fwd, __nv_bfloat16* __restrict__ wp_dg) {
  pdl_grid_sync();
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const int P = posconv_cgp(Cg);
  const long long n = static_cast<long long>(G) * P * taps * P;
  if (i >= n) return;
  const int c = i % P;             // inner (ci for fwd)
  const int j = (i / P) % taps;
  const int r = (i / (static_cast<long long>(P) * taps)) % P;  // row within group (co for fwd)
  const int g = i / (static_cast<long long>(P) * taps * P);
  float wf = 0.f, wd = 0.f;
  if (r < Cg && c < Cg) {
    // forward: row co=r, col ci=c, tap j
    wf = v[((static_cast<long long>(g) * Cg + r) * Cg + c) * taps + j] * gvec[j] * rsqrtf(static_cast<float>(norm2[j]));
    // dgrad: row ci=r, col co=c, tap jj = taps-1-j
    const int jj = taps - 1 - j;
    wd = v[((static_cast<long long>(g) * Cg + c) * Cg + r) * taps + jj] * gvec[jj] * rsqrtf(static_cast<float>(norm2[jj]));
  }
  wp_fwd[i] = __float2bfloat16_rn(wf);
  wp_dg[i] = __float2bfloat16_rn(wd);
}
// backward of weight_norm: dg[j] += dot[j]/norm_j;  dv = g/norm * dw - g*dot/norm^3 * v
__global__ void posconv_unprep_kernel(const float* __restrict__ v, const float* __restrict__ gvec,
                                      const double* __restrict__ norm2, const double* __restrict__ dot,
                                      const float* __restrict__ dwp, int D, int Cg, int taps, float* __restrict__ dv,
                                      float* __restrict__ dg) {
  pdl_grid_sync();
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const long long n = static_cast<long long>(D) * Cg * taps;
  if (i < taps) dg[i] += static_cast<float>(dot[i]) * rsqrtf(static_cast<float>(norm2[i]));
  if (i >= n) return;
  const int j = i % taps;
  const int ci = (i / taps) % Cg;
  const int co = i / (static_cast<long long>(taps) * Cg);
  const int g = co / Cg, cog = co % Cg;
  const float inv = rsqrtf(static_cast<float>(norm2[j]));
  const float dw = dwp[((static_cast<long long>(g) * Cg + cog) * taps + j) * posconv_cgp(Cg) + ci];
  dv[i] += gvec[j] * inv * dw - gvec[j] * static_cast<float>(dot[j]) * inv * inv * inv * v[i];
}

}  // namespace b200

using namespace b200;

extern "C" {

int b200s_scale_copy_f32(const float* src, float* dst, long long n, float scale, b200s_stream stream) {
  B200_CHECK_ARG(src && dst, "scale_copy_f32: null pointer");
  if (n == 0) return 0;
  B200_CHECK_CUDA(launch_pdl(scale_copy_f32_kernel, dim3(static_cast<unsigned>(ceil_div_ll(n, 256))), dim3(256), 0, static_cast<cudaStream_t>(stream), 
      src, dst, n, scale));
  B200_CHECK_LAUNCH();
  return 0;
}

int b200s_prep_linear(const float* src, int N, int K, float scale, void* dst, long long ld, void* dstT, long long ldT,
                      b200s_stream stream) {
  B200_CHECK_ARG(src && (dst || dstT), "prep_linear: null pointer");
  dim3 grid(ceil_div(K, 32), ceil_div(N, 32)), block(32, 8);
  B200_CHECK_CUDA(launch_pdl(prep_linear_kernel, dim3(grid), dim3(block), 0, static_cast<cudaStream_t>(stream), 
      src, N, K, scale, static_cast<__nv_bfloat16*>(dst), ld, static_cast<__nv_bfloat16*>(dstT), ldT));
  B200_CHECK_LAUNCH();
  return 0;
}

// descs: DEVICE array of n_descs records {const float* src; bf16* dst; bf16* dstT; int64 ld, ldT; int32 N, K, tile_begin,
// tiles_k} (56 bytes each, tiles_k = ceil(K/64), tile_begin = prefix sum of ceil(N/64)*ceil(K/64)); total_tiles = sum of all tiles.
int b200s_prep_linear_batched(const void* descs, int n_descs, int total_tiles, b200s_stream stream) {
  B200_CHECK_ARG(descs && n_descs > 0 && total_tiles > 0, "prep_linear_batched: bad arguments");
  static_assert(sizeof(PrepLinearDesc) == 56, "descriptor layout is part of the ABI");
  B200_CHECK_CUDA(launch_pdl(prep_linear_batched_kernel, dim3(total_tiles), dim3(256), 0, static_cast<cudaStream_t>(stream), 
      static_cast<const PrepLinearDesc*>(descs), n_descs));
  B200_CHECK_LAUNCH();
  return 0;
}

int b200s_prep_conv_fwd(const float* src, int Co, int Ci, int k, void* dst, b200s_stream stream) {
  B200_CHECK_ARG(src && dst, "prep_conv_fwd: null pointer");
  const long long n = static_cast<long long>(Co) * Ci * k;
  B200_CHECK_CUDA(launch_pdl(prep_conv_fwd_kernel, dim3(static_cast<unsigned>(ceil_div_ll(n, 256))), dim3(256), 0, static_cast<cudaStream_t>(stream), 
      src, Co, Ci, k, static_cast<__nv_bfloat16*>(dst)));
  B200_CHECK_LAUNCH();
  return 0;
}

int b200s_prep_conv_dgrad(const float* src, int Co, int Ci, int k, int s, int rho, void* dst, b200s_stream stream) {
  B200_CHECK_ARG(src && dst, "prep_conv_dgrad: null pointer");
  B200_CHECK_ARG(rho >= 0 && rho < s && rho < k, "prep_conv_dgrad: bad phase");
  const int nm = (k - rho + s - 1) / s;
  const long long n = static_cast<long long>(Ci) * nm * Co;
  B200_CHECK_CUDA(launch_pdl(prep_conv_dgrad_kernel, dim3(static_cast<unsigned>(ceil_div_ll(n, 256))), dim3(256), 0, static_cast<cudaStream_t>(stream), 
      src, Co, Ci, k, s, rho, nm, static_cast<__nv_bfloat16*>(dst)));
  B200_CHECK_LAUNCH();
  return 0;
}

int b200s_unprep_conv_wgrad(const float* dwk, int Co, int Ci, int k, float* dw, b200s_stream stream) {
  B200_CHECK_ARG(dwk && dw, "unprep_conv_wgrad: null pointer");
  const long long n = static_cast<long long>(Co) * Ci * k;
  B200_CHECK_CUDA(launch_pdl(unprep_conv_wgrad_kernel, dim3(static_cast<unsigned>(ceil_div_ll(n, 256))), dim3(256), 0, static_cast<cudaStream_t>(stream), 
      dwk, Co, Ci, k, dw));
  B200_CHECK_LAUNCH();
  return 0;
}

// norm2: workspace of 2 * taps floats, 8-byte aligned (holds fp64[taps]; zeroed here)
int b200s_posconv_prep(const float* weight_v, const float* weight_g, int D, int G, int taps, float* norm2, void* wp_fwd,
                       void* wp_dgrad, b200s_stream stream) {
  B200_CHECK_ARG(weight_v && weight_g && norm2 && wp_fwd && wp_dgrad, "posconv_prep: null pointer");
  B200_CHECK_ARG(taps <= 1024 && D % G == 0 && D / G <= 128, "posconv_prep: bad sizes (at most 128 channels per group)");
  const int Cg = D / G;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  B200_CHECK_ARG((reinterpret_cast<uintptr_t>(norm2) & 7u) == 0, "posconv_prep: workspace must be 8-byte aligned");
  double* n2 = reinterpret_cast<double*>(norm2);
  B200_CHECK_CUDA(cudaMemsetAsync(n2, 0, sizeof(double) * taps, st));
  B200_CHECK_CUDA(launch_pdl(posconv_tap_reduce_kernel, dim3(4 * sm_count()), dim3(((taps + 31) / 32) * 32), 0, st, weight_v,
                             static_cast<const float*>(nullptr), D, Cg, taps, n2, static_cast<double*>(nullptr)));
  B200_CHECK_LAUNCH();
  const long long n = static_cast<long long>(G) * posconv_cgp(Cg) * taps * posconv_cgp(Cg);
  B200_CHECK_CUDA(launch_pdl(posconv_prep_kernel, dim3(static_cast<unsigned>(ceil_div_ll(n, 256))), dim3(256), 0, st, 
      weight_v, weight_g, static_cast<const double*>(n2), G, Cg, taps, static_cast<__nv_bfloat16*>(wp_fwd),
      static_cast<__nv_bfloat16*>(wp_dgrad)));
  B200_CHECK_LAUNCH();
  return 0;
}

// dwp: fp32 [G, Cg, taps, Cgp] from b200s_posconv_wgrad.  work: workspace of 4 * taps floats, 8-byte aligned (fp64[2 * taps]; zeroed here).
int b200s_posconv_unprep(const float* weight_v, const float* weight_g, const float* dwp, int D, int G, int taps,
                         float* work, float* dweight_v, float* dweight_g, b200s_stream stream) {
  B200_CHECK_ARG(weight_v && weight_g && dwp && work && dweight_v && dweight_g, "posconv_unprep: null pointer");
  B200_CHECK_ARG(D % G == 0 && D / G <= 128, "posconv_unprep: bad sizes (at most 128 channels per group)");
  const int Cg = D / G;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  B200_CHECK_ARG((reinterpret_cast<uintptr_t>(work) & 7u) == 0, "posconv_unprep: workspace must be 8-byte aligned");
  double* w2 = reinterpret_cast<double*>(work);
  B200_CHECK_CUDA(cudaMemsetAsync(w2, 0, sizeof(double) * 2 * taps, st));
  B200_CHECK_CUDA(launch_pdl(posconv_tap_reduce_kernel, dim3(4 * sm_count()), dim3(((taps + 31) / 32) * 32), 0, st, weight_v, dwp, D, Cg, taps, w2,
                             w2 + taps));
  B200_CHECK_LAUNCH();
  const long long n = static_cast<long long>(D) * Cg * taps;
  B200_CHECK_CUDA(launch_pdl(posconv_unprep_kernel, dim3(static_cast<unsigned>(ceil_div_ll(n, 256))), dim3(256), 0, st, weight_v, weight_g, static_cast<const double*>(w2), static_cast<const double*>(w2 + taps),
                                                                                   dwp, D, Cg, taps, dweight_v, dweight_g));
  B200_CHECK_LAUNCH();
  return 0;
}

}  // extern "C"
