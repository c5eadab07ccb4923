// Fused attention backward with the gated relative-position bias (autograd of WavLM/modules.py:521-563): ONE tensor-core
// kernel produces dQ, dK, dV, d gate and d tab, so the probabilities are recomputed once.  wgmma + TMA (sm_90a).
//
// CTA = 128 keys of one (batch, head); it walks over the 128-row query tiles.  Two consumer warpgroups (WG w = 0, 1) and one TMA
// warp.  Per query tile i, WG w owns query rows 64 w .. 64 w + 63 for the scores and key rows 64 w .. 64 w + 63 for the dK / dV
// accumulators (registers, across the whole loop).  Everything element-wise is done on the wgmma accumulator fragments:
//   for each 64-key half hf:
//     S  = Q_i K_hf^T,  dP = dO_i V_hf^T                     wgmma m64n64k16 (64 query rows of this WG)
//     P  = exp2(S*scale*log2e + gate_i*log2e*tab[j-i] + keymask_j - lse_i);   dS = P o (dP - Delta_i) * scale
//     P, dS -> shared memory, bf16 [128 queries][128 keys] operand tiles (two 64-key blocks); gate*dS/scale -> a bf16 staging
//     tile for the d tab diagonal sums (one tile: the first half's sums are taken before the second half is staged);
//     d gate_i += sum_j dS_ij tab[j-i] (quad shuffles, one atomic per row)
//   (all 256 threads) barrier, then
//   dV += P^T dO_i, dK += dS^T Q_i     A = P / dS tile read MN-major (M = this WG's 64 keys), B = dO / Q MN-major
//   dQ_i = dS K                        A = dS read K-major (this WG's 64 queries), added to an fp32 [B,T,D] buffer with vector
//                                      reductions (one writer CTA per key tile and query element)
//   d tab[d] = sum_i gate_i dS_{i,i+d}  diagonal sums of the staged tiles, per-CTA accumulators, flushed with atomics at the end
// Dropout: the keep bit of (query i, key j) is bit i & 31 of word drop_mask[block(i), j], written by the forward kernel.
// Padding: a CTA whose 128 keys are all padded writes zero dK / dV rows and exits; query tiles that are fully padded at the end
// of the utterance are not visited (their probabilities are zero: the forward leaves lse = +inf there).
#include "../../include/unispeech_b200.h"
#include "attn_common.cuh"
#include "common.h"

#include <algorithm>

namespace b200 {

namespace {

__device__ __forceinline__ float ex2f(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ void red_add_v2(float* dst, float a, float b) {
  asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(dst), "f"(a), "f"(b) : "memory");
}

// shared-memory map (bytes from the 1024-aligned base)
constexpr int kFK = 0;             // K tile          16 KB
constexpr int kFV = 16384;         // V tile          16 KB
constexpr int kFQ = 32768;         // Q tiles, 2 stages x 16 KB
constexpr int kFDO = 65536;        // dO tiles, 2 stages x 16 KB
constexpr int kFP = 98304;         // P  : [128 queries][128 keys] as two 64-key blocks, 32 KB
constexpr int kFDS = 131072;       // dS : same layout, 32 KB
constexpr int kFW = 163840;        // gate*dS staging for the diagonal sums: one [128 queries][66] bf16 tile
constexpr int kWStride2 = 66;      // bf16 per staged row (33 words: conflict-free row writes and diagonal reads)
constexpr int kFWBytes = 128 * kWStride2 * 2;   // 16896
constexpr int kFTab = kFW + kFWBytes;            // 180736: tab slice [(N+1)*128], dtab_acc[(N+1)*128]
constexpr int kConsumers = 256;                  // two warpgroups
constexpr int kFThreads = kConsumers + 32;       // + the TMA warp
constexpr int kProdWarp = kConsumers / 32;

}  // namespace

// shared memory of the fused backward for N key tiles (with or without the relative-position bias)
static inline int attn_bwd_smem_bytes(int N, bool bias) {
  return kFTab + static_cast<int>(sizeof(float)) * ((bias ? (N + 1) * kAttnTile : 0) + (N + 1) * kAttnTile) + 1024;
}

template <bool HAS_BIAS, bool DROP>
__global__ void __launch_bounds__(kFThreads, 1) attn_bwd_fused_kernel(const __grid_constant__ CUtensorMap tm_qkv,
                                                                      const __grid_constant__ CUtensorMap tm_do,
                                                                      const __grid_constant__ AttnParams p,
                                                                      float* __restrict__ dq_acc) {
  pdl_grid_sync();
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int k0 = blockIdx.x * kAttnTile, h = blockIdx.y, b = blockIdx.z;
  const int T = p.T, D = p.D, N = p.n_tiles;

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);  // 1024-aligned, still a __shared__ pointer (LDS/STS, not generic)
  uint8_t* sK = smem + kFK;
  uint8_t* sV = smem + kFV;
  uint8_t* sQ = smem + kFQ;
  uint8_t* sDO = smem + kFDO;
  uint8_t* sP = smem + kFP;
  uint8_t* sDS = smem + kFDS;
  float* tab_s = reinterpret_cast<float*>(smem + kFTab);  // slice[l] = tab[h, l + tab_base]
  float* dtab_acc = tab_s + (HAS_BIAS ? (N + 1) * kAttnTile : 0);  // [(N+1)*128]

  __shared__ uint64_t kv_full, qdo_full[2], qdo_free[2];
  __shared__ uint32_t key_mask_s[4];  // bit j of word j>>5: key k0 + j is padded / beyond T

  // ---- padding: which of this CTA's keys are masked, and how many query tiles hold a valid query.  ONE pass over the
  // utterance's pad bytes (every thread takes a few), one block-wide reduction: the prologue pays a single global-load latency.
  __shared__ int nq_s;
  if (tid == 0) nq_s = 1;
  int NQ = N;  // query tiles to visit
  {
    bool masked = false;
    if (tid < kAttnTile) {
      const int j = k0 + tid;
      masked = (j >= T) || (p.key_pad != nullptr && p.key_pad[static_cast<long long>(b) * T + j] != 0);
      const uint32_t bal = __ballot_sync(0xffffffffu, masked);
      if (lane == 0) key_mask_s[warp] = bal;
    }
    int last_live = -1;
    if (p.key_pad != nullptr) {
      for (int i = tid; i < T; i += kFThreads)
        if (p.key_pad[static_cast<long long>(b) * T + i] == 0) last_live = i;   // increasing i: the last hit is the largest
    }
    const int n_masked = __syncthreads_count(masked);
    if (n_masked == kAttnTile) {
      // nothing attends to these keys: dK = dV = 0
      if (tid < kAttnTile && k0 + tid < T) {
        __nv_bfloat16* dst = p.dqkv + (static_cast<long long>(b) * T + k0 + tid) * (3 * D) + D + h * kHeadDim;
#pragma unroll
        for (int g = 0; g < 8; ++g) {
          *reinterpret_cast<uint4*>(dst + g * 8) = make_uint4(0u, 0u, 0u, 0u);
          *reinterpret_cast<uint4*>(dst + D + g * 8) = make_uint4(0u, 0u, 0u, 0u);
        }
      }
      return;
    }
    if (p.key_pad != nullptr) {
      if (last_live >= 0) atomicMax(&nq_s, last_live / kAttnTile + 1);
      __syncthreads();
      NQ = nq_s;
    }
  }

  if (warp == kProdWarp && lane == 0) {
    // the producer thread initialises the barriers itself and puts K, V and the first Q / dO tiles in flight right away: they
    // land while the rest of the CTA is still filling the tables (the other warps see the barriers after the __syncthreads below)
    tma_prefetch_desc(&tm_qkv);
    tma_prefetch_desc(&tm_do);
    mbar_init(&kv_full, 1);
    for (int i = 0; i < 2; ++i) {
      mbar_init(&qdo_full[i], 1);
      mbar_init(&qdo_free[i], kConsumers / 32);  // one arrival per consumer warp once its MMAs reading the stage have retired
    }
    fence_mbar_init();
    mbar_expect_tx(&kv_full, 32768);
    tma_load_4d(sK, &tm_qkv, &kv_full, D + h * kHeadDim, k0, b, 0);
    tma_load_4d(sV, &tm_qkv, &kv_full, 2 * D + h * kHeadDim, k0, b, 0);
    for (int qi = 0; qi < 2 && qi < NQ; ++qi) {
      mbar_expect_tx(&qdo_full[qi], 32768);
      tma_load_4d(sQ + qi * 16384, &tm_qkv, &qdo_full[qi], h * kHeadDim, qi * kAttnTile, b, 0);
      tma_load_4d(sDO + qi * 16384, &tm_do, &qdo_full[qi], h * kHeadDim, qi * kAttnTile, b, 0);
    }
  }

  // per-CTA tables: slice[l] = tab[h, l + base], base = k0 - (N*128-1) + (T-1); element (query i, key k0 + j) -> l = j - i + N*128-1
  const int tab_base = k0 - (N * kAttnTile - 1) + (T - 1);
  if (HAS_BIAS) {
    const int len = (N + 1) * kAttnTile;
    const float* tab_h = p.tab + static_cast<long long>(h) * (2 * T - 1);
    for (int l = tid; l < len; l += kFThreads) {
      const int gi = l + tab_base;
      tab_s[l] = (gi >= 0 && gi < 2 * T - 1) ? tab_h[gi] : 0.f;
      dtab_acc[l] = 0.f;
    }
  }
  __syncthreads();

  if (warp == kProdWarp) {
    // ================================================================== TMA producer: Q / dO stage refills
    if (lane == 0) {
      for (int qi = 2; qi < NQ; ++qi) {
        const int s = qi & 1;
        mbar_wait(&qdo_free[s], ((qi - 2) >> 1) & 1);  // the MMAs of tile qi-2 have retired
        mbar_expect_tx(&qdo_full[s], 32768);
        tma_load_4d(sQ + s * 16384, &tm_qkv, &qdo_full[s], h * kHeadDim, qi * kAttnTile, b, 0);
        tma_load_4d(sDO + s * 16384, &tm_do, &qdo_full[s], h * kHeadDim, qi * kAttnTile, b, 0);
      }
    }
  } else {
    // ==================================================================== consumer warpgroups
    const int w = warp >> 2;                 // warpgroup: query rows 64 w.. of each tile, key rows 64 w.. of dK / dV
    const int wq = warp & 3;
    const int fr = 64 * w + 16 * wq + (lane >> 2);   // first of this thread's two fragment rows (the other is fr + 8)
    const int fc = 2 * (lane & 3);                    // column of fragment element 0 inside each 8-column group
    const float sc = p.scale * kLog2e;
    const float inv_scale = 1.0f / p.scale;
    const bool any_masked = (key_mask_s[0] | key_mask_s[1] | key_mask_s[2] | key_mask_s[3]) != 0u;  // uniform over the CTA
    const long long bh = static_cast<long long>(b) * p.H + h;

    float dv_acc[32], dk_acc[32];  // written by the first tile's MMAs (scale_d = 0)

    // diagonal sums of the staged gate*dS tile of (query tile qi, key half hf).  Task (e, s): elements (i = (jj - e) & 127, jj)
    // for jj = 16 s .. 16 s + 15: diagonal jj - i = e (not wrapped, jj >= e) or e - 128 (wrapped).  The wrap point is a per-task
    // constant, so every load is base + immediate.
    auto diag_task = [&](int qi, int hf, int e, int s) {
      const uint32_t* wtile = reinterpret_cast<const uint32_t*>(smem + kFW);
      const int w0 = e - 16 * s;  // columns jj = 16 s + c with c < w0 are on the wrapped diagonal
      const uint32_t base_nw = smem_u32(wtile) + static_cast<uint32_t>((16 * s - e) * kWStride2 + 16 * s) * 2u;
      const uint32_t base_w = base_nw + static_cast<uint32_t>(kAttnTile * kWStride2 * 2);
      float acc_all = 0.f, acc_nw = 0.f;
#pragma unroll
      for (int c = 0; c < 16; ++c) {
        const bool wrapped = c < w0;
        uint32_t v16;
        asm volatile("ld.shared.u16 %0, [%1];" : "=r"(v16) : "r"((wrapped ? base_w : base_nw) + c * (kWStride2 + 1) * 2));
        const float v = __uint_as_float(v16 << 16);
        acc_all += v;
        if (!wrapped) acc_nw += v;
      }
      const int l_nw = hf * 64 - qi * kAttnTile + e + N * kAttnTile - 1;
      if (w0 < 16) atomicAdd(&dtab_acc[l_nw], acc_nw);
      if (w0 > 0) atomicAdd(&dtab_acc[l_nw - kAttnTile], acc_all - acc_nw);
    };

    for (int qi = 0; qi < NQ; ++qi) {
      const int st = qi & 1;
      // per-row scalars of this thread's two fragment rows; lse = +inf marks out-of-range queries (p = exp2(-inf) = 0)
      float r_lse[2], r_dsc[2], r_gl[2], r_gos[2];
#pragma unroll
      for (int rr = 0; rr < 2; ++rr) {
        const int i = qi * kAttnTile + fr + 8 * rr;
        float lse = INFINITY, delta = 0.f, gate = 0.f;
        if (i < T) {
          lse = p.lse[bh * T + i];
          delta = p.delta[bh * T + i];
          if (HAS_BIAS) gate = (p.gate != nullptr) ? p.gate[bh * T + i] : 1.0f;
        }
        r_lse[rr] = lse;
        r_dsc[rr] = delta * p.scale;
        r_gl[rr] = gate * kLog2e;
        r_gos[rr] = gate * inv_scale;
      }
      float dg[2] = {0.f, 0.f};
      mbar_wait(&kv_full, 0);
      mbar_wait(&qdo_full[st], (qi >> 1) & 1);
      const uint32_t aq = smem_u32(sQ + st * 16384) + w * 8192, ad = smem_u32(sDO + st * 16384) + w * 8192;

#pragma unroll 1
      for (int hf = 0; hf < 2; ++hf) {
        float s_acc[32], d_acc[32];
        const uint32_t bk = smem_u32(sK) + hf * 8192, bv = smem_u32(sV) + hf * 8192;
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < 4; ++k)
          wgmma_m64n64k16<0, 0>(s_acc, make_smem_desc_sw128(aq + k * 32, 16, 1024), make_smem_desc_sw128(bk + k * 32, 16, 1024),
                                k > 0 ? 1u : 0u);
#pragma unroll
        for (int k = 0; k < 4; ++k)
          wgmma_m64n64k16<0, 0>(d_acc, make_smem_desc_sw128(ad + k * 32, 16, 1024), make_smem_desc_sw128(bv + k * 32, 16, 1024),
                                k > 0 ? 1u : 0u);
        wgmma_commit();
        // dropout keep words of this thread's key columns (bit = query row & 31; both fragment rows are in one 32-row block)
        const uint32_t* mrow = nullptr;
        if (DROP) mrow = p.drop_mask + (bh * (4 * N) + ((qi * kAttnTile + fr) >> 5)) * (N * kAttnTile) + k0 + hf * 64 + fc;
        wgmma_wait<0>();
        uint32_t* wtile = reinterpret_cast<uint32_t*>(smem + kFW);
#pragma unroll
        for (int g = 0; g < 8; ++g) {        // 8-column group
          uint2 kw = make_uint2(0u, 0u);     // keep words of columns fc, fc + 1 of the group
          if (DROP) kw = *reinterpret_cast<const uint2*>(mrow + 8 * g);
#pragma unroll
          for (int rr = 0; rr < 2; ++rr) {   // fragment row
            const int r = fr + 8 * rr;
            const int i = qi * kAttnTile + r;
            float pr2[2], ds2[2], w2[2];
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const int idx = 4 * g + 2 * rr + e;
              const int jj = hf * 64 + 8 * g + fc + e;   // key column inside the tile
              float tb = 0.f;
              if (HAS_BIAS) tb = tab_s[jj - r + N * kAttnTile - 1 - qi * kAttnTile];
              float x = fmaf(s_acc[idx], sc, -r_lse[rr]);
              if (HAS_BIAS) x = fmaf(r_gl[rr], tb, x);
              float pr = ex2f(x);
              if (any_masked) pr = ((key_mask_s[jj >> 5] >> (jj & 31)) & 1u) ? 0.f : pr;
              float dpv = d_acc[idx];
              bool keep = true;
              if (DROP) {  // O = (P o M) V / (1-p):  dP = M o (dO V^T) / (1-p);  dV takes the dropped probabilities (scaled at the end)
                keep = (((e ? kw.y : kw.x) >> (i & 31)) & 1u) != 0u;
                dpv = keep ? dpv * p.drop_rp : 0.f;
              }
              const float ds = pr * fmaf(dpv, p.scale, -r_dsc[rr]);  // dS * scale
              pr2[e] = keep ? pr : 0.f;
              ds2[e] = ds;
              w2[e] = 0.f;
              if (HAS_BIAS) {
                dg[rr] = fmaf(ds, tb, dg[rr]);
                w2[e] = r_gos[rr] * ds;
              }
            }
            // bf16 pairs into the operand tiles (K-major SWIZZLE_128B, block hf) and the diagonal staging tile
            const int c = 8 * g + fc;  // column inside the 64-key block
            const uint32_t off = static_cast<uint32_t>(hf * 16384 + r * 128 + ((g ^ (r & 7)) << 4) + (c & 7) * 2);
            *reinterpret_cast<uint32_t*>(sP + off) = pack_bf16x2(pr2[0], pr2[1]);
            *reinterpret_cast<uint32_t*>(sDS + off) = pack_bf16x2(ds2[0], ds2[1]);
            if (HAS_BIAS) wtile[r * (kWStride2 / 2) + (c >> 1)] = pack_bf16x2(w2[0], w2[1]);
          }
        }
        if (HAS_BIAS && hf == 0) {  // the first half's diagonal sums, then the staging tile is free for the second half
          named_bar_sync(1, kConsumers);
          diag_task(qi, 0, tid & 127, tid >> 7);
          diag_task(qi, 0, tid & 127, (tid >> 7) + 2);
          named_bar_sync(1, kConsumers);
        }
      }
      if (HAS_BIAS && p.dgate != nullptr) {
#pragma unroll
        for (int rr = 0; rr < 2; ++rr) {
          float v = dg[rr];
          v += __shfl_xor_sync(0xffffffffu, v, 1);
          v += __shfl_xor_sync(0xffffffffu, v, 2);
          const int i = qi * kAttnTile + fr + 8 * rr;
          if ((lane & 3) == 0 && i < T) atomicAdd(p.dgate + bh * T + i, v * inv_scale);
        }
      }
      fence_proxy_async_smem();  // generic-proxy smem writes -> visible to the tensor core (async proxy)
      named_bar_sync(1, kConsumers);

      // ---- dV += P^T dO, dK += dS^T Q (this WG's 64 keys), dQ = dS K (this WG's 64 queries)
      {
        const uint32_t ap = smem_u32(sP) + w * 16384, ads = smem_u32(sDS) + w * 16384;
        const uint32_t bdo = smem_u32(sDO + st * 16384), bq = smem_u32(sQ + st * 16384);
        const uint32_t adq = smem_u32(sDS) + w * 8192, bk = smem_u32(sK);
        float dq[32];
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < 8; ++k)  // K = 128 queries, 16 per step
          wgmma_m64n64k16<1, 1>(dv_acc, make_smem_desc_sw128(ap + k * 2048, 16384, 1024),
                                make_smem_desc_sw128(bdo + k * 2048, 8192, 1024), (qi > 0 || k > 0) ? 1u : 0u);
#pragma unroll
        for (int k = 0; k < 8; ++k)
          wgmma_m64n64k16<1, 1>(dk_acc, make_smem_desc_sw128(ads + k * 2048, 16384, 1024),
                                make_smem_desc_sw128(bq + k * 2048, 8192, 1024), (qi > 0 || k > 0) ? 1u : 0u);
#pragma unroll
        for (int k = 0; k < 8; ++k)  // K = 128 keys: two 64-key blocks, 16 per step
          wgmma_m64n64k16<0, 1>(dq, make_smem_desc_sw128(adq + (k >> 2) * 16384 + (k & 3) * 32, 16, 1024),
                                make_smem_desc_sw128(bk + k * 2048, 8192, 1024), k > 0 ? 1u : 0u);
        wgmma_commit();
        if (HAS_BIAS) {  // the second half's diagonal sums while the MMAs run (256 threads, 2 tasks each)
          diag_task(qi, 1, tid & 127, tid >> 7);
          diag_task(qi, 1, tid & 127, (tid >> 7) + 2);
        }
        wgmma_wait<0>();
        if (lane == 0) mbar_arrive(&qdo_free[st]);
        // dQ rows of this WG -> fp32 reductions into dq_acc[b, q, h*64 + col]  (the staged dS already carries the softmax scale)
#pragma unroll
        for (int rr = 0; rr < 2; ++rr) {
          const int q = qi * kAttnTile + fr + 8 * rr;
          if (q < T) {
            float* dst = dq_acc + (static_cast<long long>(b) * T + q) * D + h * kHeadDim + fc;
#pragma unroll
            for (int g = 0; g < 8; ++g) red_add_v2(dst + 8 * g, dq[4 * g + 2 * rr], dq[4 * g + 2 * rr + 1]);
          }
        }
      }
      named_bar_sync(1, kConsumers);  // P / dS / staging tiles may be overwritten by the next tile
    }
    // ---- dK / dV rows of this WG (keys k0 + 64 w ..): bf16 pairs straight from the fragments
#pragma unroll
    for (int rr = 0; rr < 2; ++rr) {
      const int key = k0 + fr + 8 * rr;
      if (key < T) {
        __nv_bfloat16* dst = p.dqkv + (static_cast<long long>(b) * T + key) * (3 * D) + h * kHeadDim + fc;
#pragma unroll
        for (int g = 0; g < 8; ++g) {
          const float rp = DROP ? p.drop_rp : 1.0f;   // dV = (P o M)^T dO / (1-p)
          *reinterpret_cast<uint32_t*>(dst + 2 * D + 8 * g) = pack_bf16x2(dv_acc[4 * g + 2 * rr] * rp, dv_acc[4 * g + 2 * rr + 1] * rp);
          *reinterpret_cast<uint32_t*>(dst + D + 8 * g) = pack_bf16x2(dk_acc[4 * g + 2 * rr], dk_acc[4 * g + 2 * rr + 1]);
        }
      }
    }
  }

  __syncthreads();
  if (HAS_BIAS) {
    // per-CTA accumulators -> global (the relative-position table is shared by all layers: atomics)
    if (p.dtab != nullptr) {
      for (int l = tid; l < (N + 1) * kAttnTile; l += kFThreads) {
        const int gi = l + tab_base;
        const float v = dtab_acc[l];
        if (gi >= 0 && gi < 2 * T - 1 && v != 0.f) atomicAdd(p.dtab + static_cast<long long>(h) * (2 * T - 1) + gi, v);
      }
    }
  }
}

// Delta_i = sum_d dO_id O_id (fp32 [B,H,T]); also clears d gate, which the fused kernel accumulates with atomics.
__global__ void __launch_bounds__(256) attn_delta2_kernel(const __nv_bfloat16* __restrict__ o,
                                                          const __nv_bfloat16* __restrict__ dout, int B, int T, int H,
                                                          float* __restrict__ delta, float* __restrict__ dgate) {
  pdl_grid_sync();
  const int lane = threadIdx.x & 31;
  const long long row = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  if (row >= static_cast<long long>(B) * T) return;
  const int D = H * kHeadDim;
  const long long b = row / T, t = row % T;
  for (int h = 0; h < H; ++h) {
    const float2 a = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(o + row * D + h * kHeadDim + lane * 2));
    const float2 g = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(dout + row * D + h * kHeadDim + lane * 2));
    const float s = warp_sum(a.x * g.x + a.y * g.y);
    if (lane == 0) {
      delta[(b * H + h) * T + t] = s;
      if (dgate != nullptr) dgate[(b * H + h) * T + t] = 0.f;
    }
  }
}

// dq_acc (fp32 [B*T, D]) -> bf16 into the q columns of dqkv [B*T, 3D]; the accumulator is cleared for the next layer.
__global__ void __launch_bounds__(256) attn_dq_convert_kernel(float* __restrict__ dq_acc, __nv_bfloat16* __restrict__ dqkv,
                                                              long long rows, int D) {
  pdl_grid_sync();
  const int vec_per_row = D / 8;
  const long long n = rows * vec_per_row;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long row = i / vec_per_row;
    const int c = static_cast<int>(i % vec_per_row) * 8;
    float4* src = reinterpret_cast<float4*>(dq_acc + row * D + c);
    const float4 a = src[0], bq = src[1];
    uint4 w;
    w.x = pack_bf16x2(a.x, a.y); w.y = pack_bf16x2(a.z, a.w);
    w.z = pack_bf16x2(bq.x, bq.y); w.w = pack_bf16x2(bq.z, bq.w);
    *reinterpret_cast<uint4*>(dqkv + row * 3 * D + c) = w;
    src[0] = make_float4(0.f, 0.f, 0.f, 0.f);
    src[1] = make_float4(0.f, 0.f, 0.f, 0.f);
  }
}

int make_qkv_tmap(CUtensorMap* out, const void* qkv, int T, int B, int D3, int box_rows);


// Delta pre-kernel, the fused kernel and the dQ conversion on one stream (see the entry points below for the contract).
static int attn_bwd_launch(const void* qkv, const void* out, const void* dout, const float* gate, const float* tab,
                           const uint8_t* key_pad, const float* lse, float* delta, float* dq_acc, void* dqkv, float* dgate,
                           float* dtab, int B, int T, int H, float scale, float drop_p, const uint32_t* drop_mask,
                           cudaStream_t st) {
  const int D = H * kHeadDim;
  const long long rows = static_cast<long long>(B) * T;
  B200_CHECK_CUDA(launch_pdl(attn_delta2_kernel, dim3(static_cast<unsigned>(ceil_div_ll(rows * 32, 256))), dim3(256), 0, st,
      static_cast<const __nv_bfloat16*>(out), static_cast<const __nv_bfloat16*>(dout), B, T, H, delta,
      tab != nullptr ? dgate : nullptr));
  B200_CHECK_LAUNCH();

  CUtensorMap tm_qkv, tm_do;
  if (make_qkv_tmap(&tm_qkv, qkv, T, B, 3 * D, kAttnTile)) return -3;
  if (make_qkv_tmap(&tm_do, dout, T, B, D, kAttnTile)) return -3;
  AttnParams p;
  memset(&p, 0, sizeof(p));
  p.T = T; p.H = H; p.B = B; p.D = D;
  p.n_tiles = ceil_div(T, kAttnTile);
  p.scale = scale;
  p.gate = gate; p.tab = tab; p.key_pad = key_pad;
  p.lse = const_cast<float*>(lse);
  p.dout = static_cast<const __nv_bfloat16*>(dout);
  p.delta = delta;
  p.dqkv = static_cast<__nv_bfloat16*>(dqkv);
  p.dgate = dgate;
  p.dtab = dtab;
  const bool drop = drop_p > 0.f;
  p.drop_mask = const_cast<uint32_t*>(drop_mask);
  p.drop_rp = 1.0f / (1.0f - drop_p);
  const int N = p.n_tiles;
  const int smem = attn_bwd_smem_bytes(N, tab != nullptr);
  B200_CHECK_ARG(smem <= 232448 - 512, "attn_bwd: T=%d needs %d bytes of shared memory", T, smem);
  dim3 grid(N, H, B);
  void (*kern)(const CUtensorMap, const CUtensorMap, const AttnParams, float*) =
      tab != nullptr ? (drop ? attn_bwd_fused_kernel<true, true> : attn_bwd_fused_kernel<true, false>)
                     : (drop ? attn_bwd_fused_kernel<false, true> : attn_bwd_fused_kernel<false, false>);
  B200_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  B200_CHECK_CUDA(launch_pdl(kern, dim3(grid), dim3(kFThreads), smem, st, tm_qkv, tm_do, p, dq_acc));
  B200_CHECK_LAUNCH();
  const long long nvec = rows * (D / 8);
  const int blocks = static_cast<int>(std::min<long long>(ceil_div_ll(nvec, 256), static_cast<long long>(sm_count()) * 16));
  B200_CHECK_CUDA(launch_pdl(attn_dq_convert_kernel, dim3(blocks), dim3(256), 0, st, dq_acc, static_cast<__nv_bfloat16*>(dqkv), rows, D));
  B200_CHECK_LAUNCH();
  return 0;
}

}  // namespace b200

using namespace b200;

extern "C" {

// Backward of b200s_attn_fwd.  out/dout: bf16 [B,T,D]; lse from the forward; delta: fp32 [B,H,T] workspace;
// dqkv: bf16 [B,T,3D] (fully written for valid rows); dgate: fp32 [B,H,T] (written); dtab: fp32 [H,2T-1] (ACCUMULATED with
// atomics -- the caller zeroes it once per step, the table is shared by all layers).  gate/tab/dgate/dtab NULL = no bias.
// The fp32 dQ reduction buffer is allocated on the stream for the call (b200s_attn_bwd_fused takes it from the caller).
int b200s_attn_bwd(const void* qkv, const void* out, const void* dout, const float* gate, const float* tab,
                   const uint8_t* key_pad, const float* lse, float* delta, void* dqkv, float* dgate, float* dtab, int B,
                   int T, int H, float scale, b200s_stream stream) {
  B200_CHECK_ARG(qkv && out && dout && lse && delta && dqkv, "attn_bwd: null pointer");
  B200_CHECK_ARG(T >= 1 && T <= 4096, "attn_bwd: T=%d out of range (1..4096)", T);
  B200_CHECK_ARG(!tab || (dgate && dtab), "attn_bwd: bias given but dgate/dtab missing");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const size_t bytes = sizeof(float) * static_cast<size_t>(B) * T * H * kHeadDim;
  void* dq_acc = nullptr;
  B200_CHECK_CUDA(cudaMallocAsync(&dq_acc, bytes, st));
  B200_CHECK_CUDA(cudaMemsetAsync(dq_acc, 0, bytes, st));
  const int rc = attn_bwd_launch(qkv, out, dout, gate, tab, key_pad, lse, delta, static_cast<float*>(dq_acc), dqkv, dgate, dtab, B,
                                 T, H, scale, 0.f, nullptr, st);
  B200_CHECK_CUDA(cudaFreeAsync(dq_acc, st));
  return rc;
}

// Fused backward of b200s_attn_fwd.  Same contract as b200s_attn_bwd plus dq_acc: fp32 [B,T,D] workspace that must be ZERO
// on entry and is zero again on return (the q gradient is reduced there across key tiles before it is rounded to bf16).
int b200s_attn_bwd_fused_dropout(const void* qkv, const void* out, const void* dout, const float* gate, const float* tab,
                                 const uint8_t* key_pad, const float* lse, float* delta, float* dq_acc, void* dqkv,
                                 float* dgate, float* dtab, int B, int T, int H, float scale, float drop_p,
                                 const uint32_t* drop_mask, b200s_stream stream) {
  B200_CHECK_ARG(qkv && out && dout && lse && delta && dqkv && dq_acc, "attn_bwd_fused: null pointer");
  B200_CHECK_ARG(drop_p >= 0.f && drop_p < 1.f, "attn_bwd_fused: dropout p=%f out of range [0,1)", static_cast<double>(drop_p));
  B200_CHECK_ARG(drop_p == 0.f || drop_mask != nullptr, "attn_bwd_fused: dropout needs the mask written by b200s_attn_fwd_dropout");
  B200_CHECK_ARG(T >= 1 && T <= 2048, "attn_bwd_fused: T=%d out of range (1..2048)", T);
  B200_CHECK_ARG(!tab || (dgate && dtab), "attn_bwd_fused: bias given but dgate/dtab missing");
  return attn_bwd_launch(qkv, out, dout, gate, tab, key_pad, lse, delta, dq_acc, dqkv, dgate, dtab, B, T, H, scale, drop_p,
                         drop_mask, static_cast<cudaStream_t>(stream));
}

int b200s_attn_bwd_fused(const void* qkv, const void* out, const void* dout, const float* gate, const float* tab,
                         const uint8_t* key_pad, const float* lse, float* delta, float* dq_acc, void* dqkv, float* dgate,
                         float* dtab, int B, int T, int H, float scale, b200s_stream stream) {
  return b200s_attn_bwd_fused_dropout(qkv, out, dout, gate, tab, key_pad, lse, delta, dq_acc, dqkv, dgate, dtab, B, T, H, scale,
                                      0.f, nullptr, stream);
}

}  // extern "C"
