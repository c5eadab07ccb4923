// UniSpeech-SAT utterance-contrastive head (BASELINE config #4; SURVEY.md section 8f row 1, second half) around the wgmma GEMMs:
//   src/fairseq/models/unispeech_sat/unispeech_sat.py:699-758 (forward tail / compute_pred_spk), :545-557 (compute_nce with
//   replace_inf=False), :487-543 (sample_instances: index tensors drawn on the HOST with the reference's torch.randint call order),
//   src/fairseq/modules/gumbel_vector_quantizer.py:141-201 (GumbelVectorQuantizer.forward, hard codes).
//
// The reference gathers instances = y[instance_idxs] into an [N, S, Dp] tensor, concatenates the positive, takes
// torch.cosine_similarity over [N+1, S, Dp] and a binary cross entropy over [S, N+1] (about 1.2 GB of fp32 for S = 4000,
// N = 100, Dp = 768, plus the same again for autograd).  Here one warp per frame s walks its N+1 rows of y through L2 (they are
// 6 MB in total), keeps proj_s in registers, and produces the loss, the two logged statistics and d loss / d logit in one pass;
// the backward pass recomputes the dot products and scatters d y with vector reductions -- nothing of size [N, S, Dp] exists.
//   logit[s,0] = cos(proj_s, y_s) / temp,   logit[s,1+n] = cos(proj_s, y[idx[n,s]]) / temp
//   loss = mean_{s,n} BCEWithLogits(logit[s,n], target[s,n]);   target[s,0] = 1, target[s,1+n] = [instance from the same utterance]
#include <algorithm>

#include "../../include/unispeech_b200.h"
#include "common.h"
#include "dropout.cuh"
#include "ptx.cuh"

namespace b200 {

namespace {

constexpr int kMaxPerLane = 32;  // Dp <= 1024: each lane holds Dp / 32 <= 32 elements

// lane l owns elements {128 k + 4 l .. + 3}: 8-byte bf16 loads / 16-byte fp32 reductions, conflict-free and coalesced
template <typename F>
__device__ __forceinline__ void for_each_quad(int Dp, int lane, F f) {
#pragma unroll
  for (int k = 0; k < kMaxPerLane / 4; ++k) {  // constant trip count: the register arrays are indexed by compile-time constants
    const int c = k * 128 + lane * 4;
    if (c < Dp) f(k, c);
  }
}
__device__ __forceinline__ void load4(const __nv_bfloat16* p, float* v) {
  const uint2 w = *reinterpret_cast<const uint2*>(p);
  const float2 a = unpack_bf16x2(w.x), b = unpack_bf16x2(w.y);
  v[0] = a.x; v[1] = a.y; v[2] = b.x; v[3] = b.y;
}

// One warp per frame s.  g[s, n] = d loss / d logit[s, n] (fp32, already divided by S (N+1)); loss_sum += BCE sum (fp64);
// stats[0] += #{(logit >= 0) == target}, stats[1] += #{target == 1}.
__global__ void __launch_bounds__(256) sat_nce_fwd_kernel(const __nv_bfloat16* __restrict__ proj, long long p_rs,
                                                          const __nv_bfloat16* __restrict__ y, long long y_rs,
                                                          const int* __restrict__ idx, const uint8_t* __restrict__ same, int S,
                                                          int N, int Dp, float inv_temp, float* __restrict__ g,
                                                          double* __restrict__ loss_sum, int* __restrict__ stats) {
  pdl_grid_sync();
  const int lane = threadIdx.x & 31;
  const int s = (blockIdx.x * 256 + threadIdx.x) >> 5;
  if (s >= S) return;
  float pv[kMaxPerLane];
  float pp = 0.f;
  for_each_quad(Dp, lane, [&](int k, int c) {
    load4(proj + s * p_rs + c, pv + 4 * k);
#pragma unroll
    for (int e = 0; e < 4; ++e) pp = fmaf(pv[4 * k + e], pv[4 * k + e], pp);
  });
  const float pn = fmaxf(sqrtf(warp_sum(pp)), 1e-8f);  // torch.cosine_similarity clamps each norm at eps = 1e-8
  const float scale = 1.0f / (static_cast<float>(S) * static_cast<float>(N + 1));
  float lsum = 0.f;
  int n_acc = 0, n_pos = 0;
  for (int n = 0; n <= N; ++n) {
    const long long r = (n == 0) ? s : idx[static_cast<long long>(n - 1) * S + s];
    float dot = 0.f, yy = 0.f;
    for_each_quad(Dp, lane, [&](int k, int c) {
      float yv[4];
      load4(y + r * y_rs + c, yv);
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        dot = fmaf(pv[4 * k + e], yv[e], dot);
        yy = fmaf(yv[e], yv[e], yy);
      }
    });
    dot = warp_sum(dot);
    yy = warp_sum(yy);
    const float z = dot / (pn * fmaxf(sqrtf(yy), 1e-8f)) * inv_temp;
    const float t = (n == 0) ? 1.f : static_cast<float>(same[static_cast<long long>(n - 1) * S + s]);
    // BCEWithLogits: max(z, 0) - z t + log(1 + exp(-|z|));  d/dz = sigmoid(z) - t
    const float e = __expf(-fabsf(z));
    lsum += fmaxf(z, 0.f) - z * t + log1pf(e);
    const float sig = (z >= 0.f) ? 1.0f / (1.0f + e) : e / (1.0f + e);
    if (lane == 0) g[static_cast<long long>(s) * (N + 1) + n] = (sig - t) * scale;
    n_acc += ((z >= 0.f) == (t > 0.5f)) ? 1 : 0;
    n_pos += (t > 0.5f) ? 1 : 0;
  }
  if (lane == 0) {
    atomicAdd(loss_sum, static_cast<double>(lsum) * static_cast<double>(scale));
    atomicAdd(stats, n_acc);
    atomicAdd(stats + 1, n_pos);
  }
}

// wav2vec 2.0 InfoNCE on the same operands (src/fairseq/models/wav2vec/wav2vec2.py:533-553 compute_preds, criterions/
// wav2vec_criterion.py:57-62, 103-118): logit[s,0] = cos(x_s, y_s)/temp, logit[s,1+n] = cos(x_s, y[idx[n*S+s]])/temp, a negative that
// EQUALS the positive (all Dp entries: frequent with quantised targets) is masked with -inf; loss += sum_s (logsumexp_n - logit[s,0]);
// g[s,n] = softmax_n - [n == 0] (sum reduction: the criterion's sample_size divides later); stats[0] += #{argmax == 0 and not also
// argmin == 0}, stats[1] += S.  One warp per frame; the logits of a frame are parked in its g row between the two passes.
__global__ void __launch_bounds__(256) w2v_nce_fwd_kernel(const __nv_bfloat16* __restrict__ proj, long long p_rs,
                                                          const __nv_bfloat16* __restrict__ y, long long y_rs,
                                                          const int* __restrict__ idx, int S, int N, int Dp, float inv_temp,
                                                          float* __restrict__ g, double* __restrict__ loss_sum,
                                                          int* __restrict__ stats) {
  pdl_grid_sync();
  const int lane = threadIdx.x & 31;
  const int s = (blockIdx.x * 256 + threadIdx.x) >> 5;
  if (s >= S) return;
  float pv[kMaxPerLane], py[kMaxPerLane];
  float pp = 0.f;
  for_each_quad(Dp, lane, [&](int k, int c) {
    load4(proj + s * p_rs + c, pv + 4 * k);
    load4(y + s * y_rs + c, py + 4 * k);
#pragma unroll
    for (int e = 0; e < 4; ++e) pp = fmaf(pv[4 * k + e], pv[4 * k + e], pp);
  });
  const float pn = fmaxf(sqrtf(warp_sum(pp)), 1e-8f);
  float* grow = g + static_cast<long long>(s) * (N + 1);
  float zmax = -INFINITY, z0 = 0.f, zmin_others = INFINITY, zmax_others = -INFINITY;
  for (int n = 0; n <= N; ++n) {
    const long long r = (n == 0) ? s : idx[static_cast<long long>(n - 1) * S + s];
    float dot = 0.f, yy = 0.f;
    bool eq = true;
    for_each_quad(Dp, lane, [&](int k, int c) {
      float yv[4];
      load4(y + r * y_rs + c, yv);
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        dot = fmaf(pv[4 * k + e], yv[e], dot);
        yy = fmaf(yv[e], yv[e], yy);
        eq = eq && (yv[e] == py[4 * k + e]);
      }
    });
    dot = warp_sum(dot);
    yy = warp_sum(yy);
    eq = __all_sync(0xffffffffu, eq);
    float z = dot / (pn * fmaxf(sqrtf(yy), 1e-8f)) * inv_temp;
    if (n == 0) {
      z0 = z;
    } else {
      if (eq) z = -INFINITY;  // neg_is_pos
      zmin_others = fminf(zmin_others, z);
      zmax_others = fmaxf(zmax_others, z);
    }
    zmax = fmaxf(zmax, z);
    if (lane == 0) grow[n] = z;
  }
  __syncwarp();
  float esum = 0.f;
  for (int n = lane; n <= N; n += 32) esum += __expf(grow[n] - zmax);
  esum = warp_sum(esum);
  const float inv = 1.0f / esum;
  for (int n = lane; n <= N; n += 32) grow[n] = __expf(grow[n] - zmax) * inv - (n == 0 ? 1.f : 0.f);
  if (lane == 0) {
    atomicAdd(loss_sum, static_cast<double>(logf(esum) + zmax - z0));
    const bool is_max = (N == 0) || (z0 >= zmax_others), is_min = (N == 0) || (z0 <= zmin_others);
    atomicAdd(stats, (is_max && !is_min) ? 1 : 0);
    atomicAdd(stats + 1, 1);
  }
}

// Backward: dacc[r, :] (fp32 [S, Dp], += with vector reductions) receives d loss / d y_r; d loss / d proj_s goes to dacc[s, :]
// when proj IS y (no quantizer: `y = proj_x`, unispeech_sat.py:707-709), else to dproj_acc[s, :].  up = upstream gradient of the
// loss scalar (DEVICE float).
__global__ void __launch_bounds__(256) sat_nce_bwd_kernel(const __nv_bfloat16* __restrict__ proj, long long p_rs,
                                                          const __nv_bfloat16* __restrict__ y, long long y_rs,
                                                          const int* __restrict__ idx, int S, int N, int Dp, float inv_temp,
                                                          const float* __restrict__ g, const float* __restrict__ up,
                                                          float* __restrict__ dproj_acc, float* __restrict__ dy_acc) {
  pdl_grid_sync();
  const int lane = threadIdx.x & 31;
  const int s = (blockIdx.x * 256 + threadIdx.x) >> 5;
  if (s >= S) return;
  const float upv = *up;
  float pv[kMaxPerLane], dp[kMaxPerLane];
  float pp = 0.f;
  for_each_quad(Dp, lane, [&](int k, int c) {
    load4(proj + s * p_rs + c, pv + 4 * k);
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      pp = fmaf(pv[4 * k + e], pv[4 * k + e], pp);
      dp[4 * k + e] = 0.f;
    }
  });
  const float pn = fmaxf(sqrtf(warp_sum(pp)), 1e-8f);
  const float ipn = 1.0f / pn;
  for (int n = 0; n <= N; ++n) {
    const long long r = (n == 0) ? s : idx[static_cast<long long>(n - 1) * S + s];
    float yv[kMaxPerLane];
    float dot = 0.f, yy = 0.f;
    for_each_quad(Dp, lane, [&](int k, int c) {
      load4(y + r * y_rs + c, yv + 4 * k);
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        dot = fmaf(pv[4 * k + e], yv[4 * k + e], dot);
        yy = fmaf(yv[4 * k + e], yv[4 * k + e], yy);
      }
    });
    dot = warp_sum(dot);
    yy = warp_sum(yy);
    const float yn = fmaxf(sqrtf(yy), 1e-8f);
    const float iyn = 1.0f / yn;
    const float c = dot * ipn * iyn;                                             // cosine
    const float gz = g[static_cast<long long>(s) * (N + 1) + n] * upv * inv_temp;  // d loss / d cos
    // d cos / d p = y / (|p||y|) - cos p / |p|^2;   d cos / d y = p / (|p||y|) - cos y / |y|^2
    const float a = gz * ipn * iyn, bp = gz * c * ipn * ipn, by = gz * c * iyn * iyn;
    float* dst = dy_acc + r * static_cast<long long>(Dp);
    for_each_quad(Dp, lane, [&](int k, int cc) {
      float d4[4];
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        dp[4 * k + e] += a * yv[4 * k + e] - bp * pv[4 * k + e];
        d4[e] = a * pv[4 * k + e] - by * yv[4 * k + e];
      }
      asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(dst + cc), "f"(d4[0]), "f"(d4[1]), "f"(d4[2]), "f"(d4[3])
                   : "memory");
    });
  }
  float* dst = dproj_acc + static_cast<long long>(s) * Dp;
  for_each_quad(Dp, lane, [&](int k, int cc) {
    asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(dst + cc), "f"(dp[4 * k]), "f"(dp[4 * k + 1]),
                 "f"(dp[4 * k + 2]), "f"(dp[4 * k + 3])
                 : "memory");
  });
}

// fp32 [rows, N] -> bf16 [rows, N] (row strides in elements)
__global__ void __launch_bounds__(256) f32_to_bf16_rows_kernel(const float* __restrict__ src, long long s_rs,
                                                               __nv_bfloat16* __restrict__ dst, long long d_rs, long long rows,
                                                               int N) {
  pdl_grid_sync();
  const int vpr = N >> 2;
  const long long total = rows * vpr;
  for (long long v = static_cast<long long>(blockIdx.x) * 256 + threadIdx.x; v < total; v += static_cast<long long>(gridDim.x) * 256) {
    const long long r = v / vpr;
    const int c = static_cast<int>(v - r * vpr) << 2;
    const float4 a = *reinterpret_cast<const float4*>(src + r * s_rs + c);
    uint2 w;
    w.x = pack_bf16x2(a.x, a.y);
    w.y = pack_bf16x2(a.z, a.w);
    *reinterpret_cast<uint2*>(dst + r * d_rs + c) = w;
  }
}

// Gumbel(0,1) sample of element `ctr` from the counter-based hash of dropout.cuh: u = (bits + 0.5) / 2^32 in (0,1), g = -log(-log u).
// (F.gumbel_softmax draws -log(Exponential(1)) from torch's Philox stream, which no other implementation reproduces; the oracle
// restates THIS generator, exactly like the dropout masks.)  The accurate logf, not __logf: __logf's error near 1 is absolute
// (up to 2^-21.4), while -log u there is as small as 6e-8, so the largest noise values -- the ones that pick the code and
// dominate the soft sample's gradient -- would be off by percents.
__device__ __forceinline__ float gumbel_noise(uint32_t k0, uint32_t k1, uint32_t ctr) {
  const float u = (static_cast<float>(drop_bits(k0, k1, ctr)) + 0.5f) * 2.3283064365386963e-10f;
  return -logf(-logf(fminf(u, 0.99999994f)));
}

// ---------------------------------------------------------------- Gumbel vector quantizer, hard codes
// One warp per (frame s, group grp): logits[s, grp*V .. +V) (bf16 GEMM output of weight_proj).  code = argmax_v (first maximum,
// like torch.max); q[s, grp*dv .. +dv) = vars[grp*V + code, :] (bf16).  Statistics for the two logged perplexities: counts[grp, v]
// += [v == code] and probs[grp, v] += softmax(logits)_v, accumulated per block in shared memory first.
// Training mode (gumbel != 0): the code is argmax_v (logit_v + Gumbel noise) = the hard sample of F.gumbel_softmax(hard=True); the
// logged statistics keep using the noise-free logits, as in the reference (gumbel_vector_quantizer.py:152-170).
__global__ void __launch_bounds__(256) vq_hard_kernel(const __nv_bfloat16* __restrict__ logits, long long l_rs,
                                                      const float* __restrict__ vars, int S, int G, int V, int dv,
                                                      int* __restrict__ codes, __nv_bfloat16* __restrict__ q, long long q_rs,
                                                      float* __restrict__ counts, float* __restrict__ probs, int gumbel,
                                                      uint32_t k0, uint32_t k1) {
  pdl_grid_sync();
  extern __shared__ float sm[];  // [2][G*V]
  float* s_cnt = sm;
  float* s_prob = sm + G * V;
  for (int i = threadIdx.x; i < 2 * G * V; i += 256) sm[i] = 0.f;
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const long long warps = (static_cast<long long>(gridDim.x) * 256) >> 5;
  for (long long w = (static_cast<long long>(blockIdx.x) * 256 + threadIdx.x) >> 5; w < static_cast<long long>(S) * G; w += warps) {
    const int s = static_cast<int>(w / G), grp = static_cast<int>(w % G);
    const __nv_bfloat16* row = logits + s * l_rs + grp * V;
    // carg: arg-max of the NOISE-FREE logits (the logged hard_probs / code_perplexity use it in both modes,
    // gumbel_vector_quantizer.py:152-163); arg: arg-max that selects the code (with Gumbel noise in training mode)
    float mx = -INFINITY, hmx = -INFINITY;
    int carg = 0x7fffffff, arg = 0x7fffffff;
    for (int v = lane; v < V; v += 32) {
      const float x = __bfloat162float(row[v]);
      if (x > mx) { mx = x; carg = v; }
      const float xs = gumbel ? x + gumbel_noise(k0, k1, static_cast<uint32_t>(w) * static_cast<uint32_t>(V) + v) : x;
      if (xs > hmx) { hmx = xs; arg = v; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float om = __shfl_xor_sync(0xffffffffu, mx, o);
      const int oc = __shfl_xor_sync(0xffffffffu, carg, o);
      if (om > mx || (om == mx && oc < carg)) { mx = om; carg = oc; }
      const float oh = __shfl_xor_sync(0xffffffffu, hmx, o);
      const int oa = __shfl_xor_sync(0xffffffffu, arg, o);
      if (oh > hmx || (oh == hmx && oa < arg)) { hmx = oh; arg = oa; }
    }
    float sum = 0.f;
    for (int v = lane; v < V; v += 32) sum += __expf(__bfloat162float(row[v]) - mx);
    sum = warp_sum(sum);
    const float rs = 1.0f / sum;
    for (int v = lane; v < V; v += 32) atomicAdd(&s_prob[grp * V + v], __expf(__bfloat162float(row[v]) - mx) * rs);
    if (lane == 0) {
      atomicAdd(&s_cnt[grp * V + carg], 1.0f);
      codes[w] = arg;
    }
    const float* src = vars + (static_cast<long long>(grp) * V + arg) * dv;
    for (int d = lane; d < dv; d += 32) q[s * q_rs + grp * dv + d] = __float2bfloat16_rn(src[d]);
  }
  __syncthreads();
  for (int i = threadIdx.x; i < G * V; i += 256) {
    if (s_cnt[i] != 0.f) atomicAdd(&counts[i], s_cnt[i]);
    atomicAdd(&probs[i], s_prob[i]);
  }
}

// dvars[grp*V + code[s,grp], :] += dq[s, grp*dv .. +dv)      (backward of the codebook lookup; hard codes carry no other gradient)
__global__ void __launch_bounds__(256) vq_dvars_kernel(const __nv_bfloat16* __restrict__ dq, long long q_rs,
                                                       const int* __restrict__ codes, int S, int G, int V, int dv,
                                                       float* __restrict__ dvars) {
  pdl_grid_sync();
  const int lane = threadIdx.x & 31;
  const long long warps = (static_cast<long long>(gridDim.x) * 256) >> 5;
  for (long long w = (static_cast<long long>(blockIdx.x) * 256 + threadIdx.x) >> 5; w < static_cast<long long>(S) * G; w += warps) {
    const int s = static_cast<int>(w / G), grp = static_cast<int>(w % G);
    float* dst = dvars + (static_cast<long long>(grp) * V + codes[w]) * dv;
    for (int d = lane; d < dv; d += 32) atomicAdd(dst + d, __bfloat162float(dq[s * q_rs + grp * dv + d]));
  }
}

// d loss / d logits of the quantizer's weight_proj output (bf16 [S, G*V], written in full):
//   (a) diversity term: the criterion adds coef * (num_vars - prob_perplexity) / num_vars, prob_perplexity = sum_g exp(H(avg_p_g)),
//       avg_p_g = mean_s softmax(logits[s,g,:]) (gumbel_vector_quantizer.py:164-169, unispeech_sat.py:815-820).  With
//       c[g,v] = d loss / d avg_p[g,v] (fp32 [G*V], computed by the caller from the accumulated sums):
//           d logits[s,g,v] += p_sv (c_gv - sum_u c_gu p_su) / S
//   (b) training mode: straight-through gradient of F.gumbel_softmax(hard=True): with ys = softmax((logits + noise) / tau) and
//       h[s,g,v] = d loss / d onehot[s,g,v] = dq[s,g,:] . vars[g,v,:] (a GEMM, bf16 [S, G*V]):
//           d logits[s,g,v] += ys_v (h_v - sum_u h_u ys_u) / tau
__global__ void __launch_bounds__(256) vq_logits_bwd_kernel(const __nv_bfloat16* __restrict__ logits, long long l_rs, int S, int G,
                                                            int V, const float* __restrict__ c, const __nv_bfloat16* __restrict__ h,
                                                            long long h_rs, float inv_tau, uint32_t k0, uint32_t k1,
                                                            __nv_bfloat16* __restrict__ dlogits, long long d_rs) {
  pdl_grid_sync();
  const int lane = threadIdx.x & 31;
  const long long warps = (static_cast<long long>(gridDim.x) * 256) >> 5;
  const float inv_s = 1.0f / static_cast<float>(S);
  for (long long w = (static_cast<long long>(blockIdx.x) * 256 + threadIdx.x) >> 5; w < static_cast<long long>(S) * G; w += warps) {
    const int s = static_cast<int>(w / G), grp = static_cast<int>(w % G);
    const __nv_bfloat16* row = logits + s * l_rs + grp * V;
    // softmax statistics of the noise-free logits (a) and of (logits + noise) / tau (b)
    float mx = -INFINITY, mxs = -INFINITY;
    for (int v = lane; v < V; v += 32) {
      const float x = __bfloat162float(row[v]);
      mx = fmaxf(mx, x);
      if (h != nullptr) mxs = fmaxf(mxs, (x + gumbel_noise(k0, k1, static_cast<uint32_t>(w) * static_cast<uint32_t>(V) + v)) * inv_tau);
    }
    mx = warp_max(mx);
    if (h != nullptr) mxs = warp_max(mxs);
    float sum = 0.f, sums = 0.f, cdot = 0.f, hdot = 0.f;
    for (int v = lane; v < V; v += 32) {
      const float x = __bfloat162float(row[v]);
      const float e = __expf(x - mx);
      sum += e;
      if (c != nullptr) cdot = fmaf(c[grp * V + v], e, cdot);
      if (h != nullptr) {
        const float es = __expf((x + gumbel_noise(k0, k1, static_cast<uint32_t>(w) * static_cast<uint32_t>(V) + v)) * inv_tau - mxs);
        sums += es;
        hdot = fmaf(__bfloat162float(h[s * h_rs + grp * V + v]), es, hdot);
      }
    }
    sum = warp_sum(sum);
    cdot = warp_sum(cdot) / sum;
    if (h != nullptr) {
      sums = warp_sum(sums);
      hdot = warp_sum(hdot) / sums;
    }
    for (int v = lane; v < V; v += 32) {
      const float x = __bfloat162float(row[v]);
      float d = 0.f;
      if (c != nullptr) d = __expf(x - mx) / sum * (c[grp * V + v] - cdot) * inv_s;
      if (h != nullptr) {
        const float ys = __expf((x + gumbel_noise(k0, k1, static_cast<uint32_t>(w) * static_cast<uint32_t>(V) + v)) * inv_tau - mxs) / sums;
        d += ys * (__bfloat162float(h[s * h_rs + grp * V + v]) - hdot) * inv_tau;
      }
      dlogits[s * d_rs + grp * V + v] = __float2bfloat16_rn(d);
    }
  }
}

}  // namespace

}  // namespace b200

using namespace b200;

extern "C" {

int b200s_sat_nce_fwd(const void* proj, long long proj_rs, const void* y, long long y_rs, const int* idx, const uint8_t* same, int S,
                      int N, int Dp, float logit_temp, float* g, double* loss_sum, int* stats, b200s_stream stream) {
  B200_CHECK_ARG(proj && y && g && loss_sum && stats, "sat_nce_fwd: null pointer");
  B200_CHECK_ARG(N == 0 || (idx && same), "sat_nce_fwd: instances need their indices and same-utterance flags");
  B200_CHECK_ARG(Dp > 0 && Dp % 4 == 0 && Dp <= 1024, "sat_nce_fwd: Dp=%d must be a multiple of 4, <= 1024", Dp);
  B200_CHECK_ARG(proj_rs % 4 == 0 && y_rs % 4 == 0, "sat_nce_fwd: row strides must be multiples of 4 elements");
  B200_CHECK_ARG(logit_temp > 0.f, "sat_nce_fwd: logit_temp must be positive");
  if (S == 0) return 0;
  B200_CHECK_CUDA(launch_pdl(sat_nce_fwd_kernel, dim3(ceil_div(S, 8)), dim3(256), 0, static_cast<cudaStream_t>(stream),
                             static_cast<const __nv_bfloat16*>(proj), proj_rs, static_cast<const __nv_bfloat16*>(y), y_rs, idx,
                             same, S, N, Dp, 1.0f / logit_temp, g, loss_sum, stats));
  B200_CHECK_LAUNCH();
  return 0;
}

int b200s_w2v_nce_fwd(const void* proj, long long proj_rs, const void* y, long long y_rs, const int* idx, int S, int N, int Dp,
                      float logit_temp, float* g, double* loss_sum, int* stats, b200s_stream stream) {
  B200_CHECK_ARG(proj && y && g && loss_sum && stats, "w2v_nce_fwd: null pointer");
  B200_CHECK_ARG(N == 0 || idx, "w2v_nce_fwd: negatives need their indices");
  B200_CHECK_ARG(Dp > 0 && Dp % 4 == 0 && Dp <= 1024, "w2v_nce_fwd: Dp=%d must be a multiple of 4, <= 1024", Dp);
  B200_CHECK_ARG(proj_rs % 4 == 0 && y_rs % 4 == 0, "w2v_nce_fwd: row strides must be multiples of 4 elements");
  B200_CHECK_ARG(logit_temp > 0.f, "w2v_nce_fwd: logit_temp must be positive");
  if (S == 0) return 0;
  B200_CHECK_CUDA(launch_pdl(w2v_nce_fwd_kernel, dim3(ceil_div(S, 8)), dim3(256), 0, static_cast<cudaStream_t>(stream),
                             static_cast<const __nv_bfloat16*>(proj), proj_rs, static_cast<const __nv_bfloat16*>(y), y_rs, idx, S, N,
                             Dp, 1.0f / logit_temp, g, loss_sum, stats));
  B200_CHECK_LAUNCH();
  return 0;
}

int b200s_sat_nce_bwd(const void* proj, long long proj_rs, const void* y, long long y_rs, const int* idx, int S, int N, int Dp,
                      float logit_temp, const float* g, const float* upstream, float* dproj_acc, float* dy_acc,
                      b200s_stream stream) {
  B200_CHECK_ARG(proj && y && g && upstream && dproj_acc && dy_acc, "sat_nce_bwd: null pointer");
  B200_CHECK_ARG(N == 0 || idx, "sat_nce_bwd: instances need their indices");
  B200_CHECK_ARG(Dp > 0 && Dp % 4 == 0 && Dp <= 1024, "sat_nce_bwd: Dp=%d must be a multiple of 4, <= 1024", Dp);
  B200_CHECK_ARG(proj_rs % 4 == 0 && y_rs % 4 == 0, "sat_nce_bwd: row strides must be multiples of 4 elements");
  if (S == 0) return 0;
  B200_CHECK_CUDA(launch_pdl(sat_nce_bwd_kernel, dim3(ceil_div(S, 8)), dim3(256), 0, static_cast<cudaStream_t>(stream),
                             static_cast<const __nv_bfloat16*>(proj), proj_rs, static_cast<const __nv_bfloat16*>(y), y_rs, idx, S,
                             N, Dp, 1.0f / logit_temp, g, upstream, dproj_acc, dy_acc));
  B200_CHECK_LAUNCH();
  return 0;
}

int b200s_f32_to_bf16_rows(const float* src, long long src_rs, void* dst, long long dst_rs, long long rows, int N,
                           b200s_stream stream) {
  B200_CHECK_ARG(src && dst, "f32_to_bf16_rows: null pointer");
  B200_CHECK_ARG(N > 0 && N % 4 == 0 && src_rs % 4 == 0 && dst_rs % 4 == 0, "f32_to_bf16_rows: N and strides must be multiples of 4");
  if (rows == 0) return 0;
  const int grid = static_cast<int>(std::min<long long>(ceil_div_ll(rows * (N / 4), 256), 16LL * sm_count()));
  B200_CHECK_CUDA(launch_pdl(f32_to_bf16_rows_kernel, dim3(grid), dim3(256), 0, static_cast<cudaStream_t>(stream), src, src_rs,
                             static_cast<__nv_bfloat16*>(dst), dst_rs, rows, N));
  B200_CHECK_LAUNCH();
  return 0;
}

int b200s_vq_hard(const void* logits, long long logits_rs, const float* vars, int S, int G, int V, int dv, int* codes, void* q,
                  long long q_rs, float* counts, float* probs, int gumbel, uint32_t key0, uint32_t key1, b200s_stream stream) {
  B200_CHECK_ARG(logits && vars && codes && q && counts && probs, "vq_hard: null pointer");
  B200_CHECK_ARG(G > 0 && V > 0 && dv > 0 && 2 * G * V * 4 <= 96 * 1024, "vq_hard: G=%d x V=%d does not fit the block accumulators", G, V);
  B200_CHECK_ARG(static_cast<long long>(S) * G * V < (1LL << 32), "vq_hard: S*G*V exceeds the 32-bit noise counter");
  if (S == 0) return 0;
  const int grid = static_cast<int>(std::min<long long>(ceil_div_ll(static_cast<long long>(S) * G, 8), 2LL * sm_count()));
  const int smem = 2 * G * V * 4;
  B200_CHECK_CUDA(cudaFuncSetAttribute(vq_hard_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  B200_CHECK_CUDA(launch_pdl(vq_hard_kernel, dim3(grid), dim3(256), smem, static_cast<cudaStream_t>(stream),
                             static_cast<const __nv_bfloat16*>(logits), logits_rs, vars, S, G, V, dv, codes,
                             static_cast<__nv_bfloat16*>(q), q_rs, counts, probs, gumbel, key0, key1));
  B200_CHECK_LAUNCH();
  return 0;
}

int b200s_vq_logits_bwd(const void* logits, long long logits_rs, int S, int G, int V, const float* c, const void* h, long long h_rs,
                        float tau, uint32_t key0, uint32_t key1, void* dlogits, long long dlogits_rs, b200s_stream stream) {
  B200_CHECK_ARG(logits && dlogits, "vq_logits_bwd: null pointer");
  B200_CHECK_ARG(h == nullptr || tau > 0.f, "vq_logits_bwd: tau must be positive");
  if (S == 0) return 0;
  const int grid = static_cast<int>(std::min<long long>(ceil_div_ll(static_cast<long long>(S) * G, 8), 8LL * sm_count()));
  B200_CHECK_CUDA(launch_pdl(vq_logits_bwd_kernel, dim3(grid), dim3(256), 0, static_cast<cudaStream_t>(stream),
                             static_cast<const __nv_bfloat16*>(logits), logits_rs, S, G, V, c, static_cast<const __nv_bfloat16*>(h),
                             h_rs, h != nullptr ? 1.0f / tau : 0.f, key0, key1, static_cast<__nv_bfloat16*>(dlogits), dlogits_rs));
  B200_CHECK_LAUNCH();
  return 0;
}

int b200s_vq_dvars(const void* dq, long long dq_rs, const int* codes, int S, int G, int V, int dv, float* dvars,
                   b200s_stream stream) {
  B200_CHECK_ARG(dq && codes && dvars, "vq_dvars: null pointer");
  if (S == 0) return 0;
  const int grid = static_cast<int>(std::min<long long>(ceil_div_ll(static_cast<long long>(S) * G, 8), 8LL * sm_count()));
  B200_CHECK_CUDA(launch_pdl(vq_dvars_kernel, dim3(grid), dim3(256), 0, static_cast<cudaStream_t>(stream),
                             static_cast<const __nv_bfloat16*>(dq), dq_rs, codes, S, G, V, dv, dvars));
  B200_CHECK_LAUNCH();
  return 0;
}

}  // extern "C"
