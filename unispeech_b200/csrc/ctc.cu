// CTC fine-tuning loss (Graves et al. 2006; the `ctc` criterion of the reference, src/fairseq/criterions/ctc.py) on the bf16
// logits of the fine-tuning wrappers' `proj` head, log-softmax included.  Log-probabilities are never materialised: a warp-per-
// frame kernel writes lse[t] = logsumexp_c logit[t,c] and everything below uses lp[t,c] = logit[t,c] - lse[t].
//
//   alpha kernel  (the loss)      alpha_t(s) = lp[t,l'_s] + LSE(alpha_{t-1}(s), alpha_{t-1}(s-1), alpha_{t-1}(s-2) if l'_s != blank, != l'_{s-2})
//   beta  kernel  (the gradient)  beta_t(s)  = lp[t,l'_s] + LSE(beta_{t+1}(s),  beta_{t+1}(s+1),  beta_{t+1}(s+2)  if l'_{s+2} != blank, != l'_s)
//                                 gamma_t(s) = exp(alpha_t(s) + beta_t(s) - lp[t,l'_s] + nll)        in [0,1], sums to 1 over s
//                                 d nll / d logit[t,c] = softmax(logit[t,:])_c - sum_{s: l'_s = c} gamma_t(s)
// over the extended label sequence l' = (blank, l_1, blank, ..., l_S, blank).  Each is one CTA per utterance with one thread per
// position of l', the state double-buffered in shared memory and ONE barrier per frame: a serial chain of input_len steps, bound
// by the latency of a step.  So nothing a step needs comes straight from global memory: every thread loads its own label's logit,
// lse and (beta kernel) log_alpha into registers kPre frames ahead of the frame that consumes them.  (Streaming the utterance's
// rows into a shared-memory ring with bulk copies was measured against this and was slower -- 2.47 vs 1.72 ms for forward +
// backward at B = 8, T = 999, V = 32 on an H100 80GB HBM3 with a 700 W power limit -- so it is not kept.)
#include <limits.h>
#include <math.h>

#include <algorithm>

#include "../../include/unispeech_b200.h"
#include "common.h"
#include "ptx.cuh"

namespace b200 {

namespace {

constexpr int kMaxV = 1024;
constexpr int kMaxExt = 2 * B200S_CTC_MAX_TARGET + 1;  // positions of l' = threads of a CTA (1023)
constexpr int kPre = 4;                                // register prefetch distance in frames

__device__ __forceinline__ float bf(const __nv_bfloat16* p) { return __bfloat162float(*p); }

// One warp per valid frame: online log-sum-exp over the V logits and the first class holding the maximum.
__global__ void __launch_bounds__(256) ctc_stats_kernel(const __nv_bfloat16* __restrict__ x, long long fs, long long bs,
                                                        const int* __restrict__ input_len, int B, int T, int V,
                                                        float* __restrict__ lse, int* __restrict__ argmax) {
  pdl_grid_sync();
  const int lane = threadIdx.x & 31;
  const long long row = (static_cast<long long>(blockIdx.x) * 256 + threadIdx.x) >> 5;
  if (row >= static_cast<long long>(B) * T) return;
  const int b = static_cast<int>(row / T), t = static_cast<int>(row - static_cast<long long>(b) * T);
  if (t >= min(max(input_len[b], 0), T)) return;
  const __nv_bfloat16* p = x + b * bs + t * fs;
  float m = -INFINITY, sum = 0.f;
  int am = INT_MAX;
  for (int c = lane; c < V; c += 32) {
    const float v = bf(p + c);
    if (v > m) {
      sum = sum * expf(m - v) + 1.f;
      m = v;
      am = c;
    } else {
      sum += expf(v - m);
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float mo = __shfl_xor_sync(0xffffffffu, m, o), so = __shfl_xor_sync(0xffffffffu, sum, o);
    const int ao = __shfl_xor_sync(0xffffffffu, am, o);
    const float mn = fmaxf(m, mo);
    // a lane without classes (V < 32) holds (-inf, 0): its term is 0 * exp(-inf) = 0
    sum = (m == mn ? sum : sum * expf(m - mn)) + (mo == mn ? so : so * expf(mo - mn));
    if (mo > m || (mo == m && ao < am)) am = ao;
    m = mn;
  }
  if (lane == 0) {
    lse[row] = m + logf(sum);
    if (argmax != nullptr) argmax[row] = am;
  }
}

__device__ __forceinline__ float lse3(float a0, float a1, float a2) {
  const float m = fmaxf(a0, fmaxf(a1, a2));
  if (m == -INFINITY) return -INFINITY;
  return m + __logf(__expf(a0 - m) + __expf(a1 - m) + __expf(a2 - m));
}

__global__ void __launch_bounds__(1024) ctc_alpha_kernel(const __nv_bfloat16* __restrict__ x, long long fs, long long bs,
                                                         const float* __restrict__ lse, const int* __restrict__ input_len,
                                                         const int* __restrict__ targets, int Smax,
                                                         const int* __restrict__ target_len, int T, int V, int blank,
                                                         int zero_infinity, float* __restrict__ log_alpha,
                                                         float* __restrict__ nll, double* __restrict__ loss_sum) {
  pdl_grid_sync();
  __shared__ float abuf[2][kMaxExt + 3];  // [2 + s]; the two leading entries stay -inf (s - 1, s - 2 below position 0)
  __shared__ int bad;
  const int b = blockIdx.x, s = threadIdx.x, Lmax = 2 * Smax + 1;
  const int len = min(max(input_len[b], 0), T);
  const int tl_raw = target_len[b], tl = min(max(tl_raw, 0), Smax), L = 2 * tl + 1;
  if (s == 0) bad = (tl_raw < 0 || tl_raw > Smax) ? 1 : 0;
  for (int i = s; i < 2 * (kMaxExt + 3); i += blockDim.x) (&abuf[0][0])[i] = -INFINITY;
  __syncthreads();
  int lab = blank;
  bool skip = false;
  if (s < L && (s & 1)) {
    lab = targets[static_cast<long long>(b) * Smax + (s >> 1)];
    if (lab < 0 || lab >= V) {
      bad = 1;
      lab = blank;
    }
    if (s >= 3) skip = lab != blank && lab != targets[static_cast<long long>(b) * Smax + (s >> 1) - 1];
  }
  if (s == 0) abuf[0][2] = 0.f;  // "alpha_{-1}": all mass before position 0, so frame 0 needs no special case

  __syncthreads();
  const __nv_bfloat16* x_b = x + b * bs;

  const float* lse_b = lse + static_cast<long long>(b) * T;
  float* la = log_alpha + static_cast<long long>(b) * T * Lmax;
  float q_lse[kPre], q_x[kPre];
#pragma unroll
  for (int j = 0; j < kPre; ++j) {
    q_lse[j] = j < len ? lse_b[j] : 0.f;
    q_x[j] = j < len ? bf(x_b + j * fs + lab) : 0.f;
  }
  int cur = 0;
  for (int t0 = 0; t0 < len; t0 += kPre) {
#pragma unroll
    for (int j = 0; j < kPre; ++j) {
      const int t = t0 + j;
      if (t >= len) break;
      const float lse_t = q_lse[j];
      const float xv = q_x[j];
      if (t + kPre < len) {
        q_lse[j] = lse_b[t + kPre];
        q_x[j] = bf(x_b + (t + kPre) * fs + lab);
      }
      if (s < L) {
        const float* p = &abuf[cur][2 + s];
        const float v = lse3(p[0], p[-1], skip ? p[-2] : -INFINITY) + (xv - lse_t);
        abuf[cur ^ 1][2 + s] = v;
        la[static_cast<long long>(t) * Lmax + s] = v;
      }
      __syncthreads();
      cur ^= 1;
    }
  }
  if (s == 0) {
    const float* p = &abuf[cur][2];
    float v = -lse3(p[L - 1], L > 1 ? p[L - 2] : -INFINITY, -INFINITY);
    if (bad) v = INFINITY;
    nll[b] = v;
    if (loss_sum != nullptr && !(zero_infinity && v == INFINITY)) atomicAdd(loss_sum, static_cast<double>(v));
  }
}

// Threads [0, L) run the recursion; threads [grad_tid0, blockDim) write the gradient row of frame t while the recursion is
// already on frame t - 1 (grad_tid0 = 0 when the CTA has no room for extra warps: everyone then does both).
__global__ void __launch_bounds__(1024) ctc_beta_grad_kernel(const __nv_bfloat16* __restrict__ x, long long fs, long long bs,
                                                             const float* __restrict__ lse, const int* __restrict__ input_len,
                                                             const int* __restrict__ targets, int Smax,
                                                             const int* __restrict__ target_len, int T, int V, int blank,
                                                             const float* __restrict__ log_alpha,
                                                             const float* __restrict__ nll, const float* __restrict__ upstream,
                                                             __nv_bfloat16* __restrict__ g, long long g_fs, long long g_bs, int Vpad,
                                                             int grad_tid0) {
  pdl_grid_sync();
  __shared__ float bbuf[2][kMaxExt + 3];  // [s]; entries at and above L stay -inf (s + 1, s + 2 above the last position)
  __shared__ float gam[2][kMaxExt + 1];   // gamma_t of the label positions (odd s), by frame parity
  __shared__ float wpart[2][32];          // per-warp sums of gamma_t over the blank positions (even s), by frame parity
  __shared__ int labs[B200S_CTC_MAX_TARGET + 1];
  __shared__ int order[B200S_CTC_MAX_TARGET + 1];  // label positions sorted by class, ties in sequence order
  __shared__ int start[kMaxV + 2];                 // order[start[c] .. start[c+1]) are the positions of class c
  const int b = blockIdx.x, s = threadIdx.x, nthr = blockDim.x, Lmax = 2 * Smax + 1;
  const int len = min(max(input_len[b], 0), T);
  const int tl = min(max(target_len[b], 0), Smax), L = 2 * tl + 1;
  const float nllv = nll[b], up = upstream[b];
  const bool feasible = nllv < INFINITY;  // the alpha kernel also reports bad lengths / labels as +inf
  __nv_bfloat16* g_b = g + b * g_bs;
  {
    const int z0 = feasible ? len : 0;  // padded frames, or the whole infeasible utterance: exact zeros
    const long long n = static_cast<long long>(T - z0) * Vpad;
    for (long long i = s; i < n; i += nthr) {
      const int t = z0 + static_cast<int>(i / Vpad), c = static_cast<int>(i % Vpad);
      g_b[t * g_fs + c] = __float2bfloat16_rn(0.f);
    }
  }
  if (!feasible || len == 0) return;

  for (int i = s; i < 2 * (kMaxExt + 3); i += nthr) (&bbuf[0][0])[i] = -INFINITY;
  for (int c = s; c < V + 2; c += nthr) start[c] = 0;
  for (int i = s; i < tl; i += nthr) labs[i] = targets[static_cast<long long>(b) * Smax + i];
  __syncthreads();
  for (int i = s; i < tl; i += nthr) atomicAdd(&start[labs[i] + 1], 1);
  if (s == 0) bbuf[0][L - 1] = 0.f;  // "beta_{len}": all mass behind the last position
  __syncthreads();
  if (s == 0)
    for (int c = 1; c <= V; ++c) start[c] += start[c - 1];
  __syncthreads();
  for (int i = s; i < tl; i += nthr) {
    const int c = labs[i];
    int rank = 0;
    for (int j = 0; j < i; ++j) rank += labs[j] == c;
    order[start[c] + rank] = 2 * i + 1;
  }
  int lab = blank;
  bool skip = false;
  if (s < L && (s & 1)) {
    lab = labs[s >> 1];
    if (s + 2 < L) skip = labs[(s >> 1) + 1] != blank && labs[(s >> 1) + 1] != lab;
  }

  __syncthreads();
  const __nv_bfloat16* x_b = x + b * bs;

  const float* lse_b = lse + static_cast<long long>(b) * T;
  const float* la = log_alpha + static_cast<long long>(b) * T * Lmax;
  const bool rec = s < L;
  const int nwarp_rec = (L + 31) >> 5;
  float q_lse[kPre], q_x[kPre], q_a[kPre];
#pragma unroll
  for (int j = 0; j < kPre; ++j) {
    const int t = len - 1 - j;
    q_lse[j] = t >= 0 ? lse_b[t] : 0.f;
    q_a[j] = (rec && t >= 0) ? la[static_cast<long long>(t) * Lmax + s] : 0.f;
    q_x[j] = t >= 0 ? bf(x_b + t * fs + lab) : 0.f;
  }
  int cur = 0;
  for (int i0 = 0; i0 < len; i0 += kPre) {
#pragma unroll
    for (int j = 0; j < kPre; ++j) {
      const int i = i0 + j;
      if (i >= len) break;
      const int t = len - 1 - i, par = i & 1;
      const float lse_t = q_lse[j], a_t = q_a[j];
      const float xv = q_x[j];
      if (t - kPre >= 0) {
        q_lse[j] = lse_b[t - kPre];
        if (rec) q_a[j] = la[static_cast<long long>(t - kPre) * Lmax + s];
        q_x[j] = bf(x_b + (t - kPre) * fs + lab);
      }
      const __nv_bfloat16* row = x_b + t * fs;
      float gm = 0.f;
      if (rec) {
        const float* p = &bbuf[cur][s];
        const float lp = xv - lse_t;
        const float v = lse3(p[0], p[1], skip ? p[2] : -INFINITY) + lp;
        bbuf[cur ^ 1][s] = v;
        gm = __expf(a_t + v - lp + nllv);  // alpha or beta = -inf: exp(-inf) = 0
        if (s & 1) gam[par][s] = gm;
      }
      const float bl = warp_sum((rec && !(s & 1)) ? gm : 0.f);  // fixed shuffle tree: deterministic
      if ((s & 31) == 0) wpart[par][s >> 5] = bl;
      __syncthreads();
      for (int cl = s - grad_tid0; cl >= 0 && cl < Vpad; cl += nthr - grad_tid0) {
        float gr = 0.f;
        if (cl < V) {
          float occ = 0.f;
          for (int k = start[cl]; k < start[cl + 1]; ++k) occ += gam[par][order[k]];
          if (cl == blank)
            for (int w = 0; w < nwarp_rec; ++w) occ += wpart[par][w];
          gr = up * (__expf(bf(row + cl) - lse_t) - occ);
        }
        g_b[t * g_fs + cl] = __float2bfloat16_rn(gr);
      }
      cur ^= 1;
    }
  }
}

}  // namespace

}  // namespace b200

using namespace b200;

#define CTC_CHECK_COMMON(name)                                                                                                   \
  B200_CHECK_ARG(B > 0 && T > 0, name ": need B > 0 and T > 0 (B=%d T=%d)", B, T);                                               \
  B200_CHECK_ARG(V >= 1 && V <= kMaxV, name ": V=%d outside [1, %d]", V, kMaxV);                                                 \
  B200_CHECK_ARG(blank >= 0 && blank < V, name ": blank=%d outside [0, V=%d)", blank, V);                                        \
  B200_CHECK_ARG(Smax >= 0 && Smax <= B200S_CTC_MAX_TARGET, name ": Smax=%d exceeds the %d labels one CTA handles", Smax,        \
                 B200S_CTC_MAX_TARGET);                                                                                          \
  B200_CHECK_ARG(targets || Smax == 0, name ": null targets")

extern "C" {

int b200s_ctc_stats(const void* logits, long long frame_stride, long long batch_stride, const int* input_len, int B, int T, int V,
                    float* lse, int* argmax, b200s_stream stream) {
  B200_CHECK_ARG(logits && input_len && lse, "ctc_stats: null pointer");
  B200_CHECK_ARG(B > 0 && T > 0, "ctc_stats: need B > 0 and T > 0 (B=%d T=%d)", B, T);
  B200_CHECK_ARG(V >= 1 && V <= kMaxV, "ctc_stats: V=%d outside [1, %d]", V, kMaxV);
  const long long rows = static_cast<long long>(B) * T;
  B200_CHECK_CUDA(launch_pdl(ctc_stats_kernel, dim3(static_cast<unsigned>(ceil_div_ll(rows * 32, 256))), dim3(256), 0,
                             static_cast<cudaStream_t>(stream), static_cast<const __nv_bfloat16*>(logits), frame_stride,
                             batch_stride, input_len, B, T, V, lse, argmax));
  B200_CHECK_LAUNCH();
  return 0;
}

int b200s_ctc_alpha(const void* logits, long long frame_stride, long long batch_stride, const float* lse, const int* input_len,
                    const int* targets, int Smax, const int* target_len, int B, int T, int V, int blank, int zero_infinity,
                    float* log_alpha, float* nll, double* loss_sum, b200s_stream stream) {
  B200_CHECK_ARG(logits && lse && input_len && target_len && log_alpha && nll, "ctc_alpha: null pointer");
  CTC_CHECK_COMMON("ctc_alpha");
  const int threads = ceil_div(2 * Smax + 1, 32) * 32;
  B200_CHECK_CUDA(launch_pdl(ctc_alpha_kernel, dim3(B), dim3(threads), 0,
                             static_cast<cudaStream_t>(stream), static_cast<const __nv_bfloat16*>(logits), frame_stride,
                             batch_stride, lse, input_len, targets, Smax, target_len, T, V, blank, zero_infinity, log_alpha, nll,
                             loss_sum));
  B200_CHECK_LAUNCH();
  return 0;
}

int b200s_ctc_beta_grad(const void* logits, long long frame_stride, long long batch_stride, const float* lse, const int* input_len,
                        const int* targets, int Smax, const int* target_len, int B, int T, int V, int blank, const float* log_alpha,
                        const float* nll, const float* upstream, void* grad, long long grad_frame_stride,
                        long long grad_batch_stride, int Vpad, b200s_stream stream) {
  B200_CHECK_ARG(logits && lse && input_len && target_len && log_alpha && nll && upstream && grad, "ctc_beta_grad: null pointer");
  CTC_CHECK_COMMON("ctc_beta_grad");
  B200_CHECK_ARG(Vpad >= V, "ctc_beta_grad: Vpad=%d < V=%d", Vpad, V);
  const int rec = ceil_div(2 * Smax + 1, 32) * 32;
  const int gradw = std::min(8, ceil_div(Vpad, 32)) * 32;  // extra warps for the gradient rows when the CTA has room
  const int threads = rec + gradw <= 1024 ? rec + gradw : rec;
  B200_CHECK_CUDA(launch_pdl(ctc_beta_grad_kernel, dim3(B), dim3(threads), 0,
                             static_cast<cudaStream_t>(stream), static_cast<const __nv_bfloat16*>(logits), frame_stride,
                             batch_stride, lse, input_len, targets, Smax, target_len, T, V, blank, log_alpha, nll, upstream,
                             static_cast<__nv_bfloat16*>(grad), grad_frame_stride, grad_batch_stride, Vpad,
                             threads > rec ? rec : 0));
  B200_CHECK_LAUNCH();
  return 0;
}

}  // extern "C"
