// First layer of ConvFeatureExtractionModel: Conv1d(1, C, k=10, stride=5, bias=conv_bias) on the raw waveform, fused with its
// normalisation and GELU (WavLM/WavLM.py:400-426,485-504).  Cin = 1 makes this HBM-bound (20 flop per output element),
// so it is a CUDA-core kernel: one warp per output frame, each lane owns C/32 channels, weights in shared memory,
// channels-last bf16 output [B, Tpad, C].  The conv output is never stored: the backward recomputes it from the waveform
// (10 samples per frame).
//   mode GN ("default" extractor, WavLM-Base): Fp32GroupNorm(C, C) = per-(b, channel) statistics over ALL frames; its kernels
//            are in conv0_gn.cu, which derives the statistics from the waveform autocorrelation.
//   mode LN ("layer_norm" extractor, WavLM-Large): Fp32LayerNorm over channels per frame, single pass (the kernels below).
#include <algorithm>

#include "../../include/unispeech_b200.h"
#include "common.h"
#include "ptx.cuh"

namespace b200 {

constexpr int kMaxTaps = 16;

template <int C>
struct LaneMap {
  static constexpr int CPL = C / 32;             // channels per lane
  static constexpr int V = (CPL >= 4) ? 4 : CPL;  // contiguous channels per vector
  static constexpr int NG = CPL / V;              // vectors per lane
  static __device__ __forceinline__ int chan(int lane, int g, int v) { return (g * 32 + lane) * V + v; }
};

// conv[c] for this lane's channels of frame t (waveform window broadcast with shuffles)
template <int C>
__device__ __forceinline__ void conv_frame(const float* __restrict__ wav_b, long long L, int t, int k, int s,
                                           const float* __restrict__ w_s, int lane, float* acc, float* win) {
  using M = LaneMap<C>;
  const long long p = static_cast<long long>(t) * s + lane;
  const float xv = (lane < k && p < L) ? wav_b[p] : 0.f;
#pragma unroll
  for (int i = 0; i < M::CPL; ++i) acc[i] = 0.f;
#pragma unroll
  for (int j = 0; j < kMaxTaps; ++j) {
    const float xj = __shfl_sync(0xffffffffu, xv, j);
    if (win) win[j] = xj;
    if (j < k) {
#pragma unroll
      for (int g = 0; g < M::NG; ++g)
#pragma unroll
        for (int v = 0; v < M::V; ++v) acc[g * M::V + v] += xj * w_s[j * C + M::chan(lane, g, v)];
    }
  }
}

template <int C>
__device__ __forceinline__ void load_weights(const float* __restrict__ w, int k, float* w_s) {
  // w: [C, 1, k] reference layout -> w_s[j][c].  Iterate in the DESTINATION order: consecutive threads write consecutive
  // shared-memory words (the source-order loop wrote with a stride of C words: 10-way bank conflicts in every block's prologue,
  // 6.8 M conflicts per launch in the ncu capture); the 20 KB source is read strided from L2 instead.
  for (int i = threadIdx.x; i < C * k; i += blockDim.x) {
    const int j = i / C, c = i - j * C;
    w_s[i] = w[c * k + j];
  }
  __syncthreads();
}

template <int C>
__device__ __forceinline__ void store_frame(__nv_bfloat16* out, const float* v, int lane) {
  using M = LaneMap<C>;
#pragma unroll
  for (int g = 0; g < M::NG; ++g) {
    __nv_bfloat16* p = out + M::chan(lane, g, 0);
    if constexpr (M::V == 4) {
      uint2 w;
      w.x = pack_bf16x2(v[g * 4 + 0], v[g * 4 + 1]);
      w.y = pack_bf16x2(v[g * 4 + 2], v[g * 4 + 3]);
      *reinterpret_cast<uint2*>(p) = w;
    } else {
      *reinterpret_cast<uint32_t*>(p) = pack_bf16x2(v[g * 2 + 0], v[g * 2 + 1]);
    }
  }
}
template <int C>
__device__ __forceinline__ void load_frame(const __nv_bfloat16* in, float* v, int lane) {
  using M = LaneMap<C>;
#pragma unroll
  for (int g = 0; g < M::NG; ++g) {
    const __nv_bfloat16* p = in + M::chan(lane, g, 0);
    if constexpr (M::V == 4) {
      const uint2 w = *reinterpret_cast<const uint2*>(p);
      const float2 a = unpack_bf16x2(w.x), b = unpack_bf16x2(w.y);
      v[g * 4 + 0] = a.x; v[g * 4 + 1] = a.y; v[g * 4 + 2] = b.x; v[g * 4 + 3] = b.y;
    } else {
      const float2 a = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(p));
      v[g * 2 + 0] = a.x; v[g * 2 + 1] = a.y;
    }
  }
}

// conv[c] += bias[c] for this lane's channels (conv_bias=True, WavLM/WavLM.py:400-403)
template <int C>
__device__ __forceinline__ void add_bias(const float* __restrict__ bias, int lane, float* acc) {
  using M = LaneMap<C>;
#pragma unroll
  for (int g = 0; g < M::NG; ++g)
#pragma unroll
    for (int v = 0; v < M::V; ++v) acc[g * M::V + v] += bias[M::chan(lane, g, v)];
}

// block-wide reduction of per-lane channel partials (acc[CPL] per warp) into dst via atomics
template <int C, typename T>
__device__ __forceinline__ void block_channel_atomic(const float* acc, T* dst, int stride, float* red /*[8][C]*/) {
  using M = LaneMap<C>;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  __syncthreads();
#pragma unroll
  for (int g = 0; g < M::NG; ++g)
#pragma unroll
    for (int v = 0; v < M::V; ++v) red[warp * C + M::chan(lane, g, v)] = acc[g * M::V + v];
  __syncthreads();
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    float s = 0.f;
    for (int w = 0; w < nw; ++w) s += red[w * C + c];
    atomicAdd(dst + static_cast<long long>(c) * stride, static_cast<T>(s));
  }
}

// ---------------------------------------------------------------------------------------------- forward kernels
// LN over channels + GELU (writes per-frame mean / rstd)
template <int C>
__global__ void __launch_bounds__(256) conv0_fwd_kernel(const float* __restrict__ wav, long long L, int T, int k, int s,
                                                        const float* __restrict__ w, const float* __restrict__ gamma,
                                                        const float* __restrict__ beta, float* __restrict__ fmean,
                                                        float* __restrict__ frstd, __nv_bfloat16* __restrict__ out,
                                                        long long out_bs, const float* __restrict__ bias) {
  pdl_grid_sync();
  using M = LaneMap<C>;
  extern __shared__ float smem[];
  float* w_s = smem;
  load_weights<C>(w, k, w_s);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int b = blockIdx.y;
  const float* wav_b = wav + static_cast<long long>(b) * L;
  float g[M::CPL], be[M::CPL];
#pragma unroll
  for (int gi = 0; gi < M::NG; ++gi)
#pragma unroll
    for (int v = 0; v < M::V; ++v) {
      g[gi * M::V + v] = gamma[M::chan(lane, gi, v)];
      be[gi * M::V + v] = beta[M::chan(lane, gi, v)];
    }
  for (int t = blockIdx.x * 8 + warp; t < T; t += gridDim.x * 8) {
    float acc[M::CPL];
    conv_frame<C>(wav_b, L, t, k, s, w_s, lane, acc, nullptr);
    if (bias != nullptr) add_bias<C>(bias, lane, acc);
    float su = 0.f;
#pragma unroll
    for (int i = 0; i < M::CPL; ++i) su += acc[i];
    const float m = warp_sum(su) * (1.0f / C);
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < M::CPL; ++i) {
      const float d = acc[i] - m;
      q += d * d;
    }
    const float r = rsqrtf(warp_sum(q) * (1.0f / C) + 1e-5f);
#pragma unroll
    for (int i = 0; i < M::CPL; ++i) acc[i] = gelu_f((acc[i] - m) * r * g[i] + be[i]);
    if (lane == 0) {
      fmean[static_cast<long long>(b) * T + t] = m;
      frstd[static_cast<long long>(b) * T + t] = r;
    }
    store_frame<C>(out + b * out_bs + static_cast<long long>(t) * C, acc, lane);
  }
}

// ---------------------------------------------------------------------------------------------- backward kernels
// LN-mode weight gradient for taps [j0, j0+JT):  dW[c, j] += sum_{b,t} dconv[b,t,c] * wav[b, s*t + j], with dconv from the
// per-frame statistics; also accumulates dgamma / dbeta (and dbias) when j0 == 0.
template <int C, int JT>
__global__ void __launch_bounds__(256) conv0_bwd_dw_kernel(const float* __restrict__ wav, long long L, int T, int k, int s,
                                                           const float* __restrict__ w, const float* __restrict__ gamma,
                                                           const float* __restrict__ beta,
                                                           const float* __restrict__ fmean, const float* __restrict__ frstd,
                                                           const __nv_bfloat16* __restrict__ da, long long da_bs, int j0,
                                                           float* __restrict__ dw, float* __restrict__ dgamma,
                                                           float* __restrict__ dbeta, const float* __restrict__ bias,
                                                           float* __restrict__ dbias) {
  pdl_grid_sync();
  using M = LaneMap<C>;
  extern __shared__ float smem[];
  float* w_s = smem;
  float* red = smem + kMaxTaps * C;
  load_weights<C>(w, k, w_s);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int b = blockIdx.y;
  const float* wav_b = wav + static_cast<long long>(b) * L;
  float g[M::CPL], be[M::CPL];
  float ag[M::CPL], ab[M::CPL], adb[M::CPL];
  float acc_dw[JT][M::CPL];
#pragma unroll
  for (int gi = 0; gi < M::NG; ++gi)
#pragma unroll
    for (int v = 0; v < M::V; ++v) {
      const int c = M::chan(lane, gi, v);
      g[gi * M::V + v] = gamma[c];
      be[gi * M::V + v] = beta[c];
    }
#pragma unroll
  for (int i = 0; i < M::CPL; ++i) {
    ag[i] = ab[i] = adb[i] = 0.f;
#pragma unroll
    for (int j = 0; j < JT; ++j) acc_dw[j][i] = 0.f;
  }
  for (int t = blockIdx.x * 8 + warp; t < T; t += gridDim.x * 8) {
    float acc[M::CPL], d[M::CPL], win[kMaxTaps];
    conv_frame<C>(wav_b, L, t, k, s, w_s, lane, acc, win);
    load_frame<C>(da + b * da_bs + static_cast<long long>(t) * C, d, lane);
    if (bias != nullptr) add_bias<C>(bias, lane, acc);
    const float m = fmean[static_cast<long long>(b) * T + t], r = frstd[static_cast<long long>(b) * T + t];
    float q1 = 0.f, q2 = 0.f;
#pragma unroll
    for (int i = 0; i < M::CPL; ++i) {
      const float xh = (acc[i] - m) * r;
      const float dz = d[i] * gelu_grad_f(g[i] * xh + be[i]);
      ag[i] += dz * xh;
      ab[i] += dz;
      const float dxh = dz * g[i];
      acc[i] = xh;
      d[i] = dxh;
      q1 += dxh;
      q2 += dxh * xh;
    }
    q1 = warp_sum(q1) * (1.0f / C);
    q2 = warp_sum(q2) * (1.0f / C);
#pragma unroll
    for (int i = 0; i < M::CPL; ++i) {
      d[i] = r * (d[i] - q1 - acc[i] * q2);
      adb[i] += d[i];  // d bias: the tap whose input is 1
    }
#pragma unroll
    for (int j = 0; j < JT; ++j) {
      const float xj = (j0 + j < k) ? win[j0 + j] : 0.f;
#pragma unroll
      for (int i = 0; i < M::CPL; ++i) acc_dw[j][i] += d[i] * xj;
    }
  }
#pragma unroll
  for (int j = 0; j < JT; ++j)
    if (j0 + j < k) block_channel_atomic<C, float>(acc_dw[j], dw + (j0 + j), k, red);  // dw layout [C, 1, k]
  if (j0 == 0) {
    block_channel_atomic<C, float>(ag, dgamma, 1, red);
    block_channel_atomic<C, float>(ab, dbeta, 1, red);
    if (dbias != nullptr) block_channel_atomic<C, float>(adb, dbias, 1, red);
  }
}

// LayerNorm-mode backward in two light passes instead of two heavy ones.  The single-kernel form above needs 16 x 10 weight
// gradient accumulators per lane on top of the LayerNorm state, which does not fit the register file, so it ran TWICE (taps 0-4,
// taps 5-9), each time recomputing the convolution, gelu' and the LayerNorm backward of every frame (2.8 ms of a 41 ms
// WavLM-Large step).  Pass A does that work once, with few registers (two blocks per SM), leaves dconv (the gradient w.r.t. the
// raw convolution output, bf16) in a workspace -- which may be the incoming gradient buffer itself -- and reduces dgamma / dbeta.
// Pass B is a pure streaming reduction dW[c, j] += sum_t dconv[t, c] * wav[s t + j] over all taps at once.
template <int C>
__global__ void __launch_bounds__(256, 2) conv0_ln_bwd_dconv_kernel(const float* __restrict__ wav, long long L, int T, int k, int s,
                                                                    const float* __restrict__ w, const float* __restrict__ gamma,
                                                                    const float* __restrict__ beta,
                                                                    const float* __restrict__ fmean, const float* __restrict__ frstd,
                                                                    const __nv_bfloat16* da, long long da_bs, __nv_bfloat16* dconv,
                                                                    long long dc_bs, float* __restrict__ dgamma,
                                                                    float* __restrict__ dbeta, const float* __restrict__ bias) {
  pdl_grid_sync();
  using M = LaneMap<C>;
  extern __shared__ float smem[];
  float* w_s = smem;
  float* red = smem + kMaxTaps * C;
  load_weights<C>(w, k, w_s);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int b = blockIdx.y;
  const float* wav_b = wav + static_cast<long long>(b) * L;
  float g[M::CPL], be[M::CPL], ag[M::CPL], ab[M::CPL];
#pragma unroll
  for (int gi = 0; gi < M::NG; ++gi)
#pragma unroll
    for (int v = 0; v < M::V; ++v) {
      const int c = M::chan(lane, gi, v);
      g[gi * M::V + v] = gamma[c];
      be[gi * M::V + v] = beta[c];
    }
#pragma unroll
  for (int i = 0; i < M::CPL; ++i) ag[i] = ab[i] = 0.f;
  for (int t = blockIdx.x * 8 + warp; t < T; t += gridDim.x * 8) {
    float acc[M::CPL], d[M::CPL];
    conv_frame<C>(wav_b, L, t, k, s, w_s, lane, acc, nullptr);
    if (bias != nullptr) add_bias<C>(bias, lane, acc);
    load_frame<C>(da + b * da_bs + static_cast<long long>(t) * C, d, lane);
    const float m = fmean[static_cast<long long>(b) * T + t], r = frstd[static_cast<long long>(b) * T + t];
    float q1 = 0.f, q2 = 0.f;
#pragma unroll
    for (int i = 0; i < M::CPL; ++i) {
      const float xh = (acc[i] - m) * r;
      const float dz = d[i] * gelu_grad_f(g[i] * xh + be[i]);
      ag[i] += dz * xh;
      ab[i] += dz;
      const float dxh = dz * g[i];
      acc[i] = xh;
      d[i] = dxh;
      q1 += dxh;
      q2 += dxh * xh;
    }
    q1 = warp_sum(q1) * (1.0f / C);
    q2 = warp_sum(q2) * (1.0f / C);
#pragma unroll
    for (int i = 0; i < M::CPL; ++i) d[i] = r * (d[i] - q1 - acc[i] * q2);
    store_frame<C>(dconv + b * dc_bs + static_cast<long long>(t) * C, d, lane);
  }
  block_channel_atomic<C, float>(ag, dgamma, 1, red);
  block_channel_atomic<C, float>(ab, dbeta, 1, red);
}

template <int C, int K>
__global__ void __launch_bounds__(256) conv0_dw_from_dconv_kernel(const float* __restrict__ wav, long long L, int T, int k, int s,
                                                                  const __nv_bfloat16* __restrict__ dconv, long long dc_bs,
                                                                  float* __restrict__ dw, float* __restrict__ dbias) {
  pdl_grid_sync();
  using M = LaneMap<C>;
  extern __shared__ float smem[];
  float* red = smem;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int b = blockIdx.y;
  const float* wav_b = wav + static_cast<long long>(b) * L;
  float acc_dw[K][M::CPL], acc_db[M::CPL];
#pragma unroll
  for (int i = 0; i < M::CPL; ++i) {
    acc_db[i] = 0.f;
#pragma unroll
    for (int j = 0; j < K; ++j) acc_dw[j][i] = 0.f;
  }
  for (int t = blockIdx.x * 8 + warp; t < T; t += gridDim.x * 8) {
    float d[M::CPL];
    load_frame<C>(dconv + b * dc_bs + static_cast<long long>(t) * C, d, lane);
    const long long p = static_cast<long long>(t) * s + lane;
    const float xv = (lane < k && p < L) ? wav_b[p] : 0.f;
#pragma unroll
    for (int j = 0; j < K; ++j) {
      const float xj = __shfl_sync(0xffffffffu, xv, j);  // 0 for j >= k
#pragma unroll
      for (int i = 0; i < M::CPL; ++i) acc_dw[j][i] = fmaf(d[i], xj, acc_dw[j][i]);
    }
    if (dbias != nullptr) {  // the tap whose input is 1
#pragma unroll
      for (int i = 0; i < M::CPL; ++i) acc_db[i] += d[i];
    }
  }
#pragma unroll
  for (int j = 0; j < K; ++j)
    if (j < k) block_channel_atomic<C, float>(acc_dw[j], dw + j, k, red);  // dw layout [C, 1, k]
  if (dbias != nullptr) block_channel_atomic<C, float>(acc_db, dbias, 1, red);
}

int conv0_gn_stats_launch(const float* wav, long long L, int B, int T, int C, int k, int s, const float* w, double* stats,
                          cudaStream_t st);
int conv0_gn_bwd_launch(const float* wav, long long L, int B, int T, int C, int k, int s, const float* w, const float* gamma,
                        const float* beta, const double* stats, float* bstats, const void* da, long long da_bs, float* dw,
                        float* dgamma, float* dbeta, cudaStream_t st);
int conv0_gn_fwd_apply_launch(const float* wav, long long L, int B, int T, int C, int k, int s, const float* w,
                              const float* gamma, const float* beta, const double* stats, void* out, long long out_bs,
                              cudaStream_t st);

static int conv0_grid_x(int T) {
  int gx = std::min(ceil_div(T, 8 * 4), std::max(1, 4 * sm_count()));
  return std::max(gx, 1);
}

}  // namespace b200

using namespace b200;

#define DISPATCH_C(C_, ...)                                             \
  if (C_ == 512) {                                                      \
    constexpr int kC = 512;                                             \
    __VA_ARGS__                                                         \
  } else if (C_ == 64) {                                                \
    constexpr int kC = 64;                                              \
    __VA_ARGS__                                                         \
  } else {                                                              \
    set_last_error("conv0: channel count %d not supported (64 / 512)", C_); \
    return -1;                                                          \
  }

extern "C" {

// Forward.  mode 0: GroupNorm(C,C) (stats: fp64 [B*C*2 + B*128] workspace: per-(b,c) sums + waveform autocorrelation); mode 1: LayerNorm over channels
// (fmean/frstd: fp32 [B,T] outputs).  wav fp32 [B,L]; w fp32 [C,1,k]; out bf16 [B, out_bs/C rows, C].
int b200s_conv0_fwd(const float* wav, long long L, int B, int T, int C, int k, int s, const float* w, const float* gamma,
                    const float* beta, int mode, double* stats, float* fmean, float* frstd, void* out, long long out_bs,
                    const float* bias, b200s_stream stream) {
  B200_CHECK_ARG(wav && w && gamma && beta && out, "conv0_fwd: null pointer");
  B200_CHECK_ARG(k <= kMaxTaps && k >= 1, "conv0_fwd: kernel size %d > %d", k, kMaxTaps);
  B200_CHECK_ARG((mode == 0 && stats) || (mode == 1 && fmean && frstd), "conv0_fwd: missing statistics buffers");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  dim3 grid(conv0_grid_x(T), B);
  DISPATCH_C(C, {
    const size_t sm_w = sizeof(float) * kMaxTaps * kC;
    if (mode == 0) {
      // GroupNorm(C, C) normalises every (utterance, channel) over all its frames: a per-channel constant shifts that mean by
      // bias[c] and leaves the variance unchanged, so the bias cancels exactly -- it is not applied (and gets no gradient)
      if (int rc = conv0_gn_stats_launch(wav, L, B, T, kC, k, s, w, stats, st)) return rc;  // analytic, from the autocorrelation
      return conv0_gn_fwd_apply_launch(wav, L, B, T, kC, k, s, w, gamma, beta, stats, out, out_bs, st);
    } else {
      B200_CHECK_CUDA(launch_pdl(conv0_fwd_kernel<kC>, dim3(grid), dim3(256), sm_w, st, wav, L, T, k, s, w, gamma, beta, fmean, frstd,
                                 static_cast<__nv_bfloat16*>(out), out_bs, bias));
    }
    B200_CHECK_LAUNCH();
  })
  return 0;
}

// Backward: da = gradient w.r.t. the layer output (after norm + GELU), bf16 [B, rows, C].  Accumulates dw [C,1,k], dgamma,
// dbeta (fp32 atomics).  bstats: fp32 [B,C,12] workspace (mode 0, zeroed here).  The waveform receives no gradient.
// dconv_ws (mode 1, optional): bf16 workspace [B, ws_bs/C rows >= T, C] for the gradient w.r.t. the raw convolution output; it
// may alias `da` (the incoming gradient is then consumed).  With it the LayerNorm-mode backward is two light passes (see above).
int b200s_conv0_bwd_ws(const float* wav, long long L, int B, int T, int C, int k, int s, const float* w, const float* gamma,
                       const float* beta, int mode, const double* stats, float* bstats, const float* fmean,
                       const float* frstd, const void* da, long long da_bs, void* dconv_ws, long long ws_bs, float* dw,
                       float* dgamma, float* dbeta, const float* bias, float* dbias, b200s_stream stream) {
  B200_CHECK_ARG(wav && w && gamma && beta && da && dw && dgamma && dbeta, "conv0_bwd: null pointer");
  B200_CHECK_ARG(k <= kMaxTaps && k >= 1, "conv0_bwd: kernel size %d > %d", k, kMaxTaps);
  B200_CHECK_ARG((mode == 0 && stats && bstats) || (mode == 1 && fmean && frstd), "conv0_bwd: missing statistics");
  B200_CHECK_ARG(!dbias || bias, "conv0_bwd: dbias needs bias");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  dim3 grid(conv0_grid_x(T), B);
  const __nv_bfloat16* dap = static_cast<const __nv_bfloat16*>(da);
  DISPATCH_C(C, {
    const size_t sm = sizeof(float) * (kMaxTaps + 8) * kC;
    constexpr int JT = 5;
    if (mode == 0) {
      // (GroupNorm mode: the bias cancels in the forward pass, its gradient is exactly zero -- dbias is left untouched)
      if (int rc = conv0_gn_bwd_launch(wav, L, B, T, kC, k, s, w, gamma, beta, stats, bstats, da, da_bs, dw, dgamma, dbeta, st))
        return rc;
    } else if (dconv_ws != nullptr && k <= 10) {
      B200_CHECK_CUDA(cudaFuncSetAttribute(conv0_ln_bwd_dconv_kernel<kC>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                           static_cast<int>(sm)));
      B200_CHECK_CUDA(launch_pdl(conv0_ln_bwd_dconv_kernel<kC>, dim3(grid), dim3(256), sm, st, wav, L, T, k, s, w, gamma, beta, fmean,
                                 frstd, dap, da_bs, static_cast<__nv_bfloat16*>(dconv_ws), ws_bs, dgamma, dbeta, bias));
      B200_CHECK_LAUNCH();
      const size_t sm_red = sizeof(float) * 8 * kC;
      B200_CHECK_CUDA(launch_pdl(conv0_dw_from_dconv_kernel<kC, 10>, dim3(grid), dim3(256), sm_red, st, wav, L, T, k, s,
                                 static_cast<const __nv_bfloat16*>(dconv_ws), ws_bs, dw, dbias));
      B200_CHECK_LAUNCH();
    } else {
      B200_CHECK_CUDA(cudaFuncSetAttribute(conv0_bwd_dw_kernel<kC, JT>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                           static_cast<int>(sm)));
      for (int j0 = 0; j0 < k; j0 += JT) {
        B200_CHECK_CUDA(launch_pdl(conv0_bwd_dw_kernel<kC, JT>, dim3(grid), dim3(256), sm, st, wav, L, T, k, s, w, gamma, beta, fmean,
                                   frstd, dap, da_bs, j0, dw, dgamma, dbeta, bias, dbias));
        B200_CHECK_LAUNCH();
      }
    }
  })
  return 0;
}

int b200s_conv0_bwd(const float* wav, long long L, int B, int T, int C, int k, int s, const float* w, const float* gamma,
                    const float* beta, int mode, const double* stats, float* bstats, const float* fmean,
                    const float* frstd, const void* da, long long da_bs, float* dw, float* dgamma, float* dbeta,
                    const float* bias, float* dbias, b200s_stream stream) {
  return b200s_conv0_bwd_ws(wav, L, B, T, C, k, s, w, gamma, beta, mode, stats, bstats, fmean, frstd, da, da_bs, nullptr, 0, dw,
                            dgamma, dbeta, bias, dbias, stream);
}

}  // extern "C"
