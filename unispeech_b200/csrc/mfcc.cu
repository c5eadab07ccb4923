// MFCC + delta features of the HuBERT recipe's first iteration (src/examples/hubert/simple_kmeans/dump_mfcc_feature.py):
//   torchaudio.compliance.kaldi.mfcc(wav, sample_frequency=16000, use_energy=False)   (every other argument at its default)
//   -> compute_deltas twice (win_length 5, replicate padding) -> concatenation [Tm, 13 + 13 + 13].
// Per frame (25 ms = 400 samples, 10 ms = 160 sample shift, snip_edges): remove the frame mean, pre-emphasis 0.97 (the first
// sample uses itself), Povey window, zero-pad to 512, power spectrum, 23 mel triangles (20 Hz .. 8 kHz, bin 256 has weight 0),
// log with float32's epsilon as floor, orthonormal DCT-II to 13 cepstra, lifter 22.  The constants are built in each CTA's
// prologue in fp64 and rounded to fp32; the per-frame arithmetic is fp32.  No vendor FFT, no floating-point atomics: every
// output is a fixed sequence of operations, so two calls are bit-identical and an utterance's features do not depend on the
// rest of the batch.
#include <algorithm>
#include <mutex>

#include <cuda_bf16.h>

#include "../../include/unispeech_b200.h"
#include "common.h"
#include "ptx.cuh"

namespace b200 {

namespace {

constexpr int kWin = 400, kShift = 160, kFft = 512, kHalf = 256;   // samples per frame, frame shift, FFT size, complex FFT size
constexpr int kMels = 23, kCeps = 13, kCols = 39, kRowCols = 64;
constexpr int kMelSlot = 64;        // weights stored per mel filter: the widest (6.4 .. 8 kHz) covers 52 bins
constexpr int kWarps = 8, kThreads = kWarps * 32;
constexpr float kLogFloor = 1.1920929e-07f;   // float32 epsilon: the recipe runs in fp32

struct FrameSmem {
  float win[kWin];
  float2 tw256[kHalf / 2];          // exp(-2 pi i k / 256), k < 128: the complex FFT's butterflies
  float2 tw512[kHalf];              // exp(-2 pi i k / 512), k < 256: the real-FFT split step
  float melw[kMels][kMelSlot];      // weights of bins mel_lo[m] .. mel_lo[m] + mel_n[m] - 1
  int mel_lo[kMels], mel_n[kMels];
  float dct[kMels][kCeps];          // orthonormal DCT-II x lifter
  double mel_of_bin[kHalf];         // prologue scratch
  float buf[kWarps][kWin];          // per warp: the frame, then its power spectrum
  float2 z[kWarps][kHalf];          // per warp: the packed frame and its 256-point FFT
};

__host__ __device__ constexpr int frames_of(int n) { return n >= kWin ? 1 + (n - kWin) / kShift : 0; }

__device__ __forceinline__ double mel_scale(double f) { return 1127.0 * log(1.0 + f / 700.0); }

__device__ __forceinline__ float2 cmul(float2 a, float2 b) {
  return make_float2(a.x * b.x - a.y * b.y, a.x * b.y + a.y * b.x);
}

__device__ void build_constants(FrameSmem& s) {
  const int tid = threadIdx.x;
  constexpr double kPi = 3.14159265358979323846;
  for (int i = tid; i < kWin; i += kThreads)
    s.win[i] = static_cast<float>(pow(0.5 - 0.5 * cos(2.0 * kPi * i / (kWin - 1)), 0.85));
  for (int k = tid; k < kHalf / 2; k += kThreads) {
    double sn, cs;
    sincospi(-2.0 * k / kHalf, &sn, &cs);
    s.tw256[k] = make_float2(static_cast<float>(cs), static_cast<float>(sn));
  }
  for (int k = tid; k < kHalf; k += kThreads) {
    double sn, cs;
    sincospi(-2.0 * k / kFft, &sn, &cs);
    s.tw512[k] = make_float2(static_cast<float>(cs), static_cast<float>(sn));
    s.mel_of_bin[k] = mel_scale(16000.0 / kFft * k);
  }
  for (int e = tid; e < kMels * kCeps; e += kThreads) {
    const int m = e / kCeps, j = e % kCeps;
    const double d = j == 0 ? sqrt(1.0 / kMels) : sqrt(2.0 / kMels) * cos(kPi / kMels * (m + 0.5) * j);
    s.dct[m][j] = static_cast<float>(d * (1.0 + 0.5 * 22.0 * sin(kPi * j / 22.0)));
  }
  __syncthreads();
  if (tid < kMels) {
    const double lo = mel_scale(20.0), hi = mel_scale(8000.0), step = (hi - lo) / (kMels + 1);
    const double left = lo + tid * step, center = left + step, right = center + step;
    int first = -1, n = 0;
    for (int k = 0; k < kHalf; ++k) {   // bin 256 (Nyquist) has weight 0
      const double mk = s.mel_of_bin[k];
      const double w = fmax(0.0, fmin((mk - left) / (center - left), (right - mk) / (right - center)));
      if (w > 0.0 && n < kMelSlot) {
        if (first < 0) first = k;
        s.melw[tid][n++] = static_cast<float>(w);
      }
    }
    s.mel_lo[tid] = first < 0 ? 0 : first;
    s.mel_n[tid] = n;
  }
  __syncthreads();
}

// One warp per frame.  Persistent CTAs; frames past an utterance's own frame count are left to mfcc_delta_kernel (zeros).
__global__ void __launch_bounds__(kThreads) mfcc_frame_kernel(const float* __restrict__ wav, long long wav_bs, int L,
                                                               const int* __restrict__ n_samples, int B, int Tm,
                                                               float* __restrict__ feats, long long feats_bs) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  FrameSmem& s = *reinterpret_cast<FrameSmem*>(smem_raw);
  build_constants(s);   // shared memory only: overlaps the previous kernel's tail
  pdl_grid_sync();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  float* buf = s.buf[warp];
  float2* z = s.z[warp];
  const long long total = static_cast<long long>(B) * Tm;
  for (long long f = static_cast<long long>(blockIdx.x) * kWarps + warp; f < total; f += static_cast<long long>(gridDim.x) * kWarps) {
    const int b = static_cast<int>(f / Tm), t = static_cast<int>(f % Tm);
    const int n = min(max(n_samples[b], 0), L);
    if (t >= frames_of(n)) continue;
    // ---- samples, frame mean (remove_dc_offset)
    const float* x = wav + b * wav_bs + static_cast<long long>(t) * kShift;
    float v[13];
    float sum = 0.f;
#pragma unroll
    for (int j = 0; j < 13; ++j) {
      const int i = lane + 32 * j;
      v[j] = i < kWin ? x[i] : 0.f;
      sum += v[j];
    }
    const float mean = warp_sum(sum) * (1.0f / kWin);
#pragma unroll
    for (int j = 0; j < 13; ++j) {
      const int i = lane + 32 * j;
      if (i < kWin) buf[i] = v[j] - mean;
    }
    __syncwarp();
    // ---- pre-emphasis, window, zero-pad to 512; packed as z[m] = y[2m] + i y[2m+1] in bit-reversed order
    for (int m = lane; m < kHalf; m += 32) {
      float y[2];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int i = 2 * m + h;
        y[h] = i < kWin ? (buf[i] - 0.97f * buf[i > 0 ? i - 1 : 0]) * s.win[i] : 0.f;
      }
      z[__brev(static_cast<unsigned>(m)) >> 24] = make_float2(y[0], y[1]);
    }
    __syncwarp();
    // ---- 256-point complex FFT, radix 2, decimation in time
#pragma unroll 1
    for (int half = 1, tstep = kHalf / 2; half < kHalf; half *= 2, tstep /= 2) {
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const int bf = lane + 32 * q;
        const int pos = bf & (half - 1);
        const int i0 = (bf - pos) * 2 + pos, i1 = i0 + half;
        const float2 a = z[i0], c = cmul(z[i1], s.tw256[pos * tstep]);
        z[i0] = make_float2(a.x + c.x, a.y + c.y);
        z[i1] = make_float2(a.x - c.x, a.y - c.y);
      }
      __syncwarp();
    }
    // ---- split step: X[k] = E[k] + W512^k O[k], power |X[k]|^2 for k < 256 (bin 256 has no mel weight)
    for (int k = lane; k < kHalf; k += 32) {
      const float2 a = z[k], c = z[(kHalf - k) & (kHalf - 1)];
      const float2 e = make_float2(0.5f * (a.x + c.x), 0.5f * (a.y - c.y));
      const float2 o = make_float2(0.5f * (a.y + c.y), -0.5f * (a.x - c.x));   // (a - conj c) / 2i
      const float2 wo = cmul(s.tw512[k], o);
      const float re = e.x + wo.x, im = e.y + wo.y;
      buf[k] = re * re + im * im;
    }
    __syncwarp();
    // ---- mel energies (one lane per filter, bins in increasing order), log, DCT x lifter
    float le = 0.f;
    if (lane < kMels) {
      const float* p = buf + s.mel_lo[lane];
      const float* w = s.melw[lane];
      const int cnt = s.mel_n[lane];
      float e = 0.f;
      for (int k = 0; k < cnt; ++k) e = fmaf(w[k], p[k], e);
      le = logf(fmaxf(e, kLogFloor));
    }
    float c = 0.f;
#pragma unroll
    for (int m = 0; m < kMels; ++m) {
      const float lm = __shfl_sync(0xffffffffu, le, m);
      if (lane < kCeps) c = fmaf(lm, s.dct[m][lane], c);
    }
    if (lane < kCeps) feats[b * feats_bs + static_cast<long long>(t) * kCols + lane] = c;
    __syncwarp();   // buf / z are rewritten by the warp's next frame
  }
}

// One thread per (utterance, frame): delta and delta-delta of compute_deltas (win_length 5: sum_k k (c[t+k] - c[t-k]) / 10),
// each pass clamping frame indices to the utterance's own [0, Tm_b - 1]; the bf16 k-means row; zeros for padded frames.
__global__ void __launch_bounds__(256) mfcc_delta_kernel(const int* __restrict__ n_samples, int L, int B, int Tm,
                                                         float* __restrict__ feats, long long feats_bs,
                                                         __nv_bfloat16* __restrict__ rows, long long rows_bs) {
  pdl_grid_sync();
  const long long f = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (f >= static_cast<long long>(B) * Tm) return;
  const int b = static_cast<int>(f / Tm), t = static_cast<int>(f % Tm);
  const int Tb = frames_of(min(max(n_samples[b], 0), L));
  float* out = feats + b * feats_bs + static_cast<long long>(t) * kCols;
  uint4* row = rows != nullptr ? reinterpret_cast<uint4*>(rows + b * rows_bs + static_cast<long long>(t) * kRowCols) : nullptr;
  if (t >= Tb) {
    for (int j = 0; j < kCols; ++j) out[j] = 0.f;
    if (row != nullptr)
      for (int q = 0; q < kRowCols / 8; ++q) row[q] = make_uint4(0u, 0u, 0u, 0u);
    return;
  }
  const float* cb = feats + b * feats_bs;
  auto cl = [Tb](int u) { return min(max(u, 0), Tb - 1); };
  float vals[kCols];
#pragma unroll
  for (int j = 0; j < kCeps; ++j) {
    auto cep = [&](int u) { return cb[static_cast<long long>(cl(u)) * kCols + j]; };
    float d[5];
#pragma unroll
    for (int o = -2; o <= 2; ++o) {
      const int u = cl(t + o);
      d[o + 2] = ((cep(u + 1) - cep(u - 1)) + 2.f * (cep(u + 2) - cep(u - 2))) / 10.f;
    }
    // delta-delta clamps the delta's own frame indices: d[o + 2] is the delta at frame cl(t + o)
    vals[j] = cep(t);
    vals[kCeps + j] = d[2];
    vals[2 * kCeps + j] = ((d[3] - d[1]) + 2.f * (d[4] - d[0])) / 10.f;
  }
#pragma unroll
  for (int j = kCeps; j < kCols; ++j) out[j] = vals[j];
  if (row != nullptr) {
#pragma unroll
    for (int q = 0; q < kRowCols / 8; ++q) {
      __align__(16) __nv_bfloat16 h[8];
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        const int j = 8 * q + e;
        h[e] = __float2bfloat16_rn(j < kCols ? vals[j] : 0.f);
      }
      row[q] = *reinterpret_cast<const uint4*>(h);
    }
  }
}

}  // namespace
}  // namespace b200

using namespace b200;

extern "C" {

int b200s_mfcc(const float* wav, long long wav_bs, int L, const int* n_samples, int B, int Tm, float* feats, long long feats_bs,
               void* rows_bf16, long long rows_bs, b200s_stream stream) {
  B200_CHECK_ARG(wav && n_samples && feats, "mfcc: null pointer");
  B200_CHECK_ARG(B >= 1 && L >= 1, "mfcc: bad sizes (B=%d, L=%d)", B, L);
  B200_CHECK_ARG(Tm == frames_of(L), "mfcc: Tm=%d, but %d samples make %d frames", Tm, L, frames_of(L));
  B200_CHECK_ARG(wav_bs >= L, "mfcc: waveform batch stride %lld < L=%d", wav_bs, L);
  B200_CHECK_ARG(feats_bs >= static_cast<long long>(Tm) * kCols, "mfcc: feature batch stride %lld < Tm*39", feats_bs);
  B200_CHECK_ARG((reinterpret_cast<uintptr_t>(wav) & 3) == 0 && (reinterpret_cast<uintptr_t>(feats) & 3) == 0,
                 "mfcc: misaligned fp32 pointer");
  if (rows_bf16 != nullptr)
    B200_CHECK_ARG(rows_bs >= static_cast<long long>(Tm) * kRowCols && rows_bs % 8 == 0 &&
                       (reinterpret_cast<uintptr_t>(rows_bf16) & 15) == 0,
                   "mfcc: bf16 rows must be 16-byte aligned with a batch stride >= Tm*64 and a multiple of 8 (got %lld)", rows_bs);
  B200_CHECK_ARG(static_cast<long long>(B) * Tm < (1LL << 31), "mfcc: too many frames");
  if (Tm == 0) return 0;   // L < 400: no utterance has a frame
  static std::once_flag once;
  static cudaError_t attr_err = cudaSuccess;
  std::call_once(once, [] {
    attr_err = cudaFuncSetAttribute(mfcc_frame_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, sizeof(FrameSmem));
  });
  B200_CHECK_CUDA(attr_err);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int frames = B * Tm;
  const int ctas = std::min(ceil_div(frames, kWarps), 2 * sm_count());
  B200_CHECK_CUDA(launch_pdl(mfcc_frame_kernel, dim3(ctas), dim3(kThreads), sizeof(FrameSmem), st, wav, wav_bs, L, n_samples, B, Tm,
                             feats, feats_bs));
  B200_CHECK_LAUNCH();
  B200_CHECK_CUDA(launch_pdl(mfcc_delta_kernel, dim3(ceil_div(frames, 256)), dim3(256), 0, st, n_samples, L, B, Tm, feats, feats_bs,
                             static_cast<__nv_bfloat16*>(rows_bf16), rows_bs));
  B200_CHECK_LAUNCH();
  return 0;
}

}  // extern "C"
