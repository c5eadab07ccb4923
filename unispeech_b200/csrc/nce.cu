// Masked-prediction head of the WavLM / HuBERT-style pre-training loss (SURVEY.md section 8f row 1), fused around the wgmma
// GEMMs of gemm.cu.  Reference: src/fairseq/models/wavlm/wavlm.py:525-576 (final_proj, compute_pred), :426-438 (compute_nce:
// cosine similarity against the positive + every label embedding, / logit_temp, -inf where a negative equals the positive)
// and src/fairseq/criterions/wavlm_criterion.py:63-87 (sum-reduced cross entropy with the positive at index 0).
//
// The reference materialises negs = label_embs.unsqueeze(1).expand(-1, S, -1) -> torch.cosine_similarity over [C+1, S, Dp]
// (3 GB of fp32 for S = 6 k frames, C = 504, Dp = 256).  Here: softmax over {positive} U {c != target} IS the softmax over the
// C classes, so with z[s,c] = cos(proj_s, E_c) / temp the loss is CE(z[s,:], target_s) and
//     z = (proj En^T) * (1/|proj_s|) / temp            En = row-normalised label embeddings (bf16 GEMM operand)
// is one [S,Dp]x[Dp,C] tensor-core GEMM plus a warp-per-row softmax kernel that also emits the backward operand
//     G[s,c] = w (softmax(z)_c - [c == target_s]) / (|proj_s| temp)
// from which  d proj = G En - (sum_c G_sc cos_sc) proj_s/|proj_s|   and   d En = G^T proj  are two more GEMMs.
// (A negative whose embedding is bit-identical to the positive's is excluded by the reference; only c == target is handled here:
// distinct rows of a trained or randomly initialised table are never identical.)
#include <algorithm>

#include "../../include/unispeech_b200.h"
#include "common.h"
#include "ptx.cuh"

namespace b200 {

namespace {

__device__ __forceinline__ void load8(const __nv_bfloat16* p, float* v) {
  const uint4 w = *reinterpret_cast<const uint4*>(p);
  const uint32_t u[4] = {w.x, w.y, w.z, w.w};
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float2 f = unpack_bf16x2(u[i]);
    v[2 * i] = f.x;
    v[2 * i + 1] = f.y;
  }
}
__device__ __forceinline__ void store8(__nv_bfloat16* p, const float* v) {
  uint4 w;
  w.x = pack_bf16x2(v[0], v[1]); w.y = pack_bf16x2(v[2], v[3]);
  w.z = pack_bf16x2(v[4], v[5]); w.w = pack_bf16x2(v[6], v[7]);
  *reinterpret_cast<uint4*>(p) = w;
}

// out[s, :] = x[idx[s], :]                       (x[masked_indices], wavlm.py:541,558)
__global__ void __launch_bounds__(256) gather_rows_kernel(const __nv_bfloat16* __restrict__ x, long long x_rs,
                                                          const int* __restrict__ idx, int S, int D,
                                                          __nv_bfloat16* __restrict__ out, long long out_rs) {
  pdl_grid_sync();
  const int vpr = D >> 3;
  const long long total = static_cast<long long>(S) * vpr;
  for (long long v = static_cast<long long>(blockIdx.x) * 256 + threadIdx.x; v < total; v += static_cast<long long>(gridDim.x) * 256) {
    const int s = static_cast<int>(v / vpr), c = static_cast<int>(v - static_cast<long long>(s) * vpr) << 3;
    *reinterpret_cast<uint4*>(out + s * out_rs + c) = *reinterpret_cast<const uint4*>(x + idx[s] * x_rs + c);
  }
}
// dx[idx[s], :] += src[s, :]  (rows of one call are distinct: plain read-modify-write)      autograd of the gather
__global__ void __launch_bounds__(256) scatter_add_rows_kernel(const __nv_bfloat16* __restrict__ src, long long src_rs,
                                                               const int* __restrict__ idx, int S, int D,
                                                               __nv_bfloat16* __restrict__ dx, long long dx_rs) {
  pdl_grid_sync();
  const int vpr = D >> 3;
  const long long total = static_cast<long long>(S) * vpr;
  for (long long v = static_cast<long long>(blockIdx.x) * 256 + threadIdx.x; v < total; v += static_cast<long long>(gridDim.x) * 256) {
    const int s = static_cast<int>(v / vpr), c = static_cast<int>(v - static_cast<long long>(s) * vpr) << 3;
    float a[8], b[8];
    load8(src + s * src_rs + c, a);
    __nv_bfloat16* d = dx + idx[s] * dx_rs + c;
    load8(d, b);
#pragma unroll
    for (int i = 0; i < 8; ++i) a[i] += b[i];
    store8(d, a);
  }
}

// En[c,:] = E[c,:] / max(|E_c|, eps) as bf16 (rows c >= C are zero), EnT = its transpose [Dp, Cpad], invn[c] = 1/max(|E_c|, eps)
__global__ void __launch_bounds__(256) nce_prep_kernel(const float* __restrict__ E, int C, int Cpad, int Dp,
                                                       __nv_bfloat16* __restrict__ En, __nv_bfloat16* __restrict__ EnT,
                                                       float* __restrict__ invn) {
  pdl_grid_sync();
  const int lane = threadIdx.x & 31;
  const int c = (blockIdx.x * 256 + threadIdx.x) >> 5;
  if (c >= Cpad) return;
  float inv = 0.f;
  if (c < C) {
    float ss = 0.f;
    for (int d = lane; d < Dp; d += 32) {
      const float e = E[static_cast<long long>(c) * Dp + d];
      ss += e * e;
    }
    ss = warp_sum(ss);
    inv = 1.0f / fmaxf(sqrtf(ss), 1e-8f);  // torch.cosine_similarity clamps each norm at eps = 1e-8
    if (lane == 0) invn[c] = inv;
  }
  for (int d = lane; d < Dp; d += 32) {
    const __nv_bfloat16 v = __float2bfloat16_rn(c < C ? E[static_cast<long long>(c) * Dp + d] * inv : 0.f);
    En[static_cast<long long>(c) * Dp + d] = v;
    EnT[static_cast<long long>(d) * Cpad + c] = v;
  }
}

// One warp per selected frame s.  zraw[s,c] = proj_s . En_c (bf16 GEMM output).  Emits G (bf16 [S,Cpad]), pn = 1/|proj_s|,
// rvec = sum_c G_sc cos_sc, and accumulates w * CE (fp64), the number of frames whose target has the largest logit.
constexpr int kMaxVec = 4;  // Cpad <= 1024: each lane keeps <= 4 vectors of 8 logits in registers
__global__ void __launch_bounds__(256) nce_ce_kernel(const __nv_bfloat16* __restrict__ proj, long long proj_rs, int Dp,
                                                     const __nv_bfloat16* __restrict__ zraw, long long z_rs,
                                                     const int* __restrict__ target, int S, int C, int Cpad, float inv_temp,
                                                     float w, __nv_bfloat16* __restrict__ G, long long g_rs,
                                                     float* __restrict__ pn, float* __restrict__ rvec,
                                                     double* __restrict__ loss_sum, int* __restrict__ correct) {
  pdl_grid_sync();
  const int lane = threadIdx.x & 31;
  const int s = (blockIdx.x * 256 + threadIdx.x) >> 5;
  if (s >= S) return;
  float ss = 0.f;
  for (int d = lane * 8; d < Dp; d += 256) {
    float a[8];
    load8(proj + s * proj_rs + d, a);
#pragma unroll
    for (int i = 0; i < 8; ++i) ss += a[i] * a[i];
  }
  const float inv = 1.0f / fmaxf(sqrtf(warp_sum(ss)), 1e-8f);
  const float zs = inv * inv_temp;
  const int t = target[s];
  float z[kMaxVec][8];
  float mx = -INFINITY;
#pragma unroll
  for (int k = 0; k < kMaxVec; ++k) {
    const int c0 = (k * 32 + lane) * 8;
    if (c0 < Cpad) {
      load8(zraw + s * z_rs + c0, z[k]);
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        z[k][i] = (c0 + i < C) ? z[k][i] * zs : -INFINITY;
        mx = fmaxf(mx, z[k][i]);
      }
    }
  }
  mx = warp_max(mx);
  float sum = 0.f, zt = 0.f, mx_other = -INFINITY;
#pragma unroll
  for (int k = 0; k < kMaxVec; ++k) {
    const int c0 = (k * 32 + lane) * 8;
    if (c0 < Cpad) {
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        sum += __expf(z[k][i] - mx);
        if (c0 + i == t) zt = z[k][i]; else mx_other = fmaxf(mx_other, z[k][i]);
      }
    }
  }
  sum = warp_sum(sum);
  zt = warp_sum(zt);  // exactly one lane holds it
  mx_other = warp_max(mx_other);
  const float lse = mx + __logf(sum);
  const float rsum = 1.0f / sum;
  float r = 0.f;
#pragma unroll
  for (int k = 0; k < kMaxVec; ++k) {
    const int c0 = (k * 32 + lane) * 8;
    if (c0 < Cpad) {
      float g[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const float p = __expf(z[k][i] - mx) * rsum;           // 0 for the padded columns (z = -inf)
        const float gz = w * (p - ((c0 + i == t) ? 1.f : 0.f));  // d loss / d z_sc
        g[i] = gz * zs;                                          // d loss / d (proj_s . En_c) at fixed |proj_s|
        const float cosv = (c0 + i < C) ? z[k][i] * (1.0f / inv_temp) : 0.f;   // z = cos / temp
        r += g[i] * cosv;
      }
      store8(G + s * g_rs + c0, g);
    }
  }
  r = warp_sum(r);
  if (lane == 0) {
    pn[s] = inv;
    rvec[s] = r;
    atomicAdd(loss_sum, static_cast<double>(w * (lse - zt)));
    if (correct != nullptr && zt >= mx_other) atomicAdd(correct, 1);  // compute_correct: argmax == 0 (ties go to index 0)
  }
}

// dproj[s,:] = dprojA[s,:] - rvec[s] * pn[s] * proj[s,:]     (the |proj_s| normalisation's share of the gradient), in place
__global__ void __launch_bounds__(256) nce_dproj_kernel(__nv_bfloat16* __restrict__ dproj, long long d_rs,
                                                        const __nv_bfloat16* __restrict__ proj, long long p_rs, int S, int Dp,
                                                        const float* __restrict__ pn, const float* __restrict__ rvec) {
  pdl_grid_sync();
  const int vpr = Dp >> 3;
  const long long total = static_cast<long long>(S) * vpr;
  for (long long v = static_cast<long long>(blockIdx.x) * 256 + threadIdx.x; v < total; v += static_cast<long long>(gridDim.x) * 256) {
    const int s = static_cast<int>(v / vpr), c = static_cast<int>(v - static_cast<long long>(s) * vpr) << 3;
    float a[8], b[8];
    load8(dproj + s * d_rs + c, a);
    load8(proj + s * p_rs + c, b);
    const float k = rvec[s] * pn[s];
#pragma unroll
    for (int i = 0; i < 8; ++i) a[i] -= k * b[i];
    store8(dproj + s * d_rs + c, a);
  }
}

// dE[c,:] += (dEn_c - (dEn_c . En_c) En_c) / |E_c|      (backward of the row normalisation; En recomputed in fp32)
__global__ void __launch_bounds__(256) nce_dlabel_kernel(const float* __restrict__ dEn, const float* __restrict__ E,
                                                         const float* __restrict__ invn, int C, int Dp,
                                                         float* __restrict__ dE) {
  pdl_grid_sync();
  const int lane = threadIdx.x & 31;
  const int c = (blockIdx.x * 256 + threadIdx.x) >> 5;
  if (c >= C) return;
  const float inv = invn[c];
  float dot = 0.f;
  for (int d = lane; d < Dp; d += 32) dot += dEn[static_cast<long long>(c) * Dp + d] * (E[static_cast<long long>(c) * Dp + d] * inv);
  dot = warp_sum(dot);
  for (int d = lane; d < Dp; d += 32) {
    const long long o = static_cast<long long>(c) * Dp + d;
    dE[o] += (dEn[o] - dot * (E[o] * inv)) * inv;
  }
}

int vec_grid(long long vecs) {
  return static_cast<int>(std::max<long long>(1, std::min<long long>(ceil_div_ll(vecs, 256), 16LL * sm_count())));
}

}  // namespace

}  // namespace b200

using namespace b200;

extern "C" {

int b200s_gather_rows(const void* x, long long x_rs, const int* idx, int S, int D, void* out, long long out_rs,
                      b200s_stream stream) {
  B200_CHECK_ARG(x && idx && out, "gather_rows: null pointer");
  B200_CHECK_ARG(D > 0 && D % 8 == 0 && x_rs % 8 == 0 && out_rs % 8 == 0, "gather_rows: D and the row strides must be multiples of 8");
  if (S <= 0) return 0;
  B200_CHECK_CUDA(launch_pdl(gather_rows_kernel, dim3(vec_grid(static_cast<long long>(S) * (D / 8))), dim3(256), 0,
                             static_cast<cudaStream_t>(stream), static_cast<const __nv_bfloat16*>(x), x_rs, idx, S, D,
                             static_cast<__nv_bfloat16*>(out), out_rs));
  B200_CHECK_LAUNCH();
  return 0;
}

int b200s_scatter_add_rows(const void* src, long long src_rs, const int* idx, int S, int D, void* dx, long long dx_rs,
                           b200s_stream stream) {
  B200_CHECK_ARG(src && idx && dx, "scatter_add_rows: null pointer");
  B200_CHECK_ARG(D > 0 && D % 8 == 0 && src_rs % 8 == 0 && dx_rs % 8 == 0, "scatter_add_rows: D and the row strides must be multiples of 8");
  if (S <= 0) return 0;
  B200_CHECK_CUDA(launch_pdl(scatter_add_rows_kernel, dim3(vec_grid(static_cast<long long>(S) * (D / 8))), dim3(256), 0,
                             static_cast<cudaStream_t>(stream), static_cast<const __nv_bfloat16*>(src), src_rs, idx, S, D,
                             static_cast<__nv_bfloat16*>(dx), dx_rs));
  B200_CHECK_LAUNCH();
  return 0;
}

int b200s_nce_prep(const float* label_embs, int C, int Cpad, int Dp, void* en, void* en_t, float* invn, b200s_stream stream) {
  B200_CHECK_ARG(label_embs && en && en_t && invn, "nce_prep: null pointer");
  B200_CHECK_ARG(C > 0 && Cpad >= C && Cpad % 64 == 0 && Cpad <= 1024, "nce_prep: need C <= Cpad <= 1024, Cpad %% 64 == 0 (C=%d Cpad=%d)", C, Cpad);
  B200_CHECK_ARG(Dp > 0 && Dp % 64 == 0, "nce_prep: Dp=%d must be a multiple of 64", Dp);
  B200_CHECK_CUDA(launch_pdl(nce_prep_kernel, dim3(ceil_div(Cpad * 32, 256)), dim3(256), 0, static_cast<cudaStream_t>(stream),
                             label_embs, C, Cpad, Dp, static_cast<__nv_bfloat16*>(en), static_cast<__nv_bfloat16*>(en_t), invn));
  B200_CHECK_LAUNCH();
  return 0;
}

int b200s_nce_ce(const void* proj, long long proj_rs, int Dp, const void* zraw, long long z_rs, const int* target, int S, int C,
                 int Cpad, float logit_temp, float weight, void* g, long long g_rs, float* pn, float* rvec, double* loss_sum,
                 int* correct, b200s_stream stream) {
  B200_CHECK_ARG(proj && zraw && target && g && pn && rvec && loss_sum, "nce_ce: null pointer");
  B200_CHECK_ARG(C > 0 && Cpad >= C && Cpad % 8 == 0 && Cpad <= 1024, "nce_ce: need C <= Cpad <= 1024, Cpad %% 8 == 0 (C=%d Cpad=%d)", C, Cpad);
  B200_CHECK_ARG(Dp % 8 == 0 && proj_rs % 8 == 0 && z_rs % 8 == 0 && g_rs % 8 == 0, "nce_ce: Dp and the row strides must be multiples of 8");
  B200_CHECK_ARG(logit_temp > 0.f, "nce_ce: logit_temp must be positive");
  if (S <= 0) return 0;
  B200_CHECK_CUDA(launch_pdl(nce_ce_kernel, dim3(static_cast<unsigned>(ceil_div_ll(static_cast<long long>(S) * 32, 256))),
                             dim3(256), 0, static_cast<cudaStream_t>(stream), static_cast<const __nv_bfloat16*>(proj), proj_rs, Dp,
                             static_cast<const __nv_bfloat16*>(zraw), z_rs, target, S, C, Cpad, 1.0f / logit_temp, weight,
                             static_cast<__nv_bfloat16*>(g), g_rs, pn, rvec, loss_sum, correct));
  B200_CHECK_LAUNCH();
  return 0;
}

int b200s_nce_dproj(void* dproj, long long d_rs, const void* proj, long long p_rs, int S, int Dp, const float* pn,
                    const float* rvec, b200s_stream stream) {
  B200_CHECK_ARG(dproj && proj && pn && rvec, "nce_dproj: null pointer");
  B200_CHECK_ARG(Dp > 0 && Dp % 8 == 0 && d_rs % 8 == 0 && p_rs % 8 == 0, "nce_dproj: Dp and the row strides must be multiples of 8");
  if (S <= 0) return 0;
  B200_CHECK_CUDA(launch_pdl(nce_dproj_kernel, dim3(vec_grid(static_cast<long long>(S) * (Dp / 8))), dim3(256), 0,
                             static_cast<cudaStream_t>(stream), static_cast<__nv_bfloat16*>(dproj), d_rs,
                             static_cast<const __nv_bfloat16*>(proj), p_rs, S, Dp, pn, rvec));
  B200_CHECK_LAUNCH();
  return 0;
}

int b200s_nce_dlabel(const float* d_en, const float* label_embs, const float* invn, int C, int Dp, float* d_label_embs,
                     b200s_stream stream) {
  B200_CHECK_ARG(d_en && label_embs && invn && d_label_embs, "nce_dlabel: null pointer");
  B200_CHECK_ARG(C > 0 && Dp > 0, "nce_dlabel: bad sizes");
  B200_CHECK_CUDA(launch_pdl(nce_dlabel_kernel, dim3(ceil_div(C * 32, 256)), dim3(256), 0, static_cast<cudaStream_t>(stream), d_en,
                             label_embs, invn, C, Dp, d_label_embs));
  B200_CHECK_LAUNCH();
  return 0;
}

}  // extern "C"
